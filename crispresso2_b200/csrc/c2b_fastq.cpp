// c2b_fastq.cpp -- native FASTQ ingest + exact de-duplication for the engine's front end (host code, no CUDA).
//
// Replaces the Python loop of process_fastq that reads the FASTQ four lines at a time and counts identical
// sequences in variantCache (reference: CRISPResso2/CRISPRessoCORE.py:1820-1849).  Semantics kept bit for bit:
//   * text-mode universal newlines: "\n", "\r\n" and a lone "\r" all end a line;
//   * a record starts at every line that exists (even an empty one) and consumes the next three lines, present or not;
//   * the sequence is line 2 with leading/trailing ASCII whitespace removed (str.strip()); a missing line is "";
//   * unique sequences are reported in first-seen order with their multiplicities.
// Output is already in the packed layout c2b_align_batch takes (bytes + int64 offsets + int32 counts).
//
// Parallel plan: (1) split the buffer at line boundaries and index line starts per thread; (2) hash every record's
// sequence (threads over record ranges); (3) shard the hash space: shard s owns the records with hash % P == s and
// walks them in file order through an open-addressing table (full byte compare on hash match -- exact, no
// probabilistic step); (4) merge the shards' (first index, count) lists by first index.
#include "c2b200.h"
#include "c2b_fastq_int.h"

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include <algorithm>
#include <atomic>
#include <memory>
#include <chrono>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <functional>
#include <vector>

namespace {

struct Seq { const uint8_t *p; uint32_t len; };

inline bool is_space(uint8_t c) { return c == ' ' || (c >= 9 && c <= 13) || (c >= 0x1c && c <= 0x1f); }   // str.strip() on ASCII

inline uint64_t hash_bytes(const uint8_t *p, size_t n)
{
    // 64-bit multiply-xorshift over 8-byte words; only used to place keys -- equality is decided by memcmp
    uint64_t h = 0x9E3779B97F4A7C15ull ^ (n * 0xff51afd7ed558ccdull);
    while (n >= 8) {
        uint64_t w; memcpy(&w, p, 8);
        h = (h ^ w) * 0xff51afd7ed558ccdull; h ^= h >> 32;
        p += 8; n -= 8;
    }
    uint64_t w = 0;
    if (n) memcpy(&w, p, n);
    h = (h ^ w) * 0xc4ceb9fe1a85ec53ull; h ^= h >> 29;
    h *= 0x9E3779B97F4A7C15ull; h ^= h >> 32;
    return h;
}

int host_threads(size_t bytes, int asked = 0)
{
    int T = asked > 0 ? asked : (int)std::thread::hardware_concurrency();
    T = std::max(1, std::min(T, 64));
    return bytes < (4u << 20) ? 1 : T;
}

template <class F> void run_threads(int T, F fn)            // fn(t) on T threads (this one is thread 0)
{
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(fn, t);
    fn(0);
    for (auto &x : th) x.join();
}

// whole file into an uninitialised buffer, pread by all host threads (page-cache copies run at memory speed in parallel)
bool read_plain(const char *path, c2b_bytes &buf, std::string &err)
{
    int fd = open(path, O_RDONLY);
    if (fd < 0) { err = std::string("cannot open ") + path; return false; }
    struct stat st;
    if (fstat(fd, &st) != 0 || st.st_size < 0) { close(fd); err = "cannot size file"; return false; }
    const size_t n = (size_t)st.st_size;
    buf.resize(n);
    const int T = host_threads(n);
    std::atomic<bool> bad(false);
    run_threads(T, [&](int t) {
        size_t a = n * (size_t)t / T;
        const size_t b = n * (size_t)(t + 1) / T;
        while (a < b) {
            const ssize_t r = pread(fd, buf.data() + a, b - a, (off_t)a);
            if (r <= 0) { bad.store(true); return; }
            a += (size_t)r;
        }
    });
    close(fd);
    if (bad.load()) { err = "short read"; return false; }
    return true;
}

// output parts written at their offsets by all host threads
// (append: after the file's current end)
bool write_parts(const char *path, const std::vector<std::string> &parts, const std::string &tail, bool append = false)
{
    int fd = open(path, O_WRONLY | O_CREAT | (append ? 0 : O_TRUNC), 0666);
    if (fd < 0) return false;
    std::vector<size_t> off(parts.size() + 1, 0);
    if (append) { const off_t end = lseek(fd, 0, SEEK_END); if (end < 0) { close(fd); return false; } off[0] = (size_t)end; }
    for (size_t k = 0; k < parts.size(); k++) off[k + 1] = off[k] + parts[k].size();
    const size_t total = off[parts.size()] + tail.size();
    if (total && ftruncate(fd, (off_t)total) != 0) { close(fd); return false; }
    std::atomic<bool> bad(false);
    auto put = [&](const char *p, size_t n, size_t at) {
        while (n) {
            const ssize_t r = pwrite(fd, p, n, (off_t)at);
            if (r <= 0) { bad.store(true); return; }
            p += r; n -= (size_t)r; at += (size_t)r;
        }
    };
    const int T = total < (4u << 20) ? 1 : (int)parts.size();
    if (T <= 1) { for (size_t k = 0; k < parts.size(); k++) put(parts[k].data(), parts[k].size(), off[k]); }
    else run_threads(T, [&](int t) { put(parts[(size_t)t].data(), parts[(size_t)t].size(), off[(size_t)t]); });
    if (!tail.empty()) put(tail.data(), tail.size(), off[parts.size()]);
    close(fd);
    return !bad.load();
}

// Blocked gzip (BGZF: what bgzip and Illumina's converters write): every member's header carries its compressed size in a 'BC'
// extra subfield, so the members can be listed without inflating anything and inflated independently -- here by all host threads,
// each member straight to its place in the output (the ISIZE trailers give the offsets).  Returns false without touching `buf`
// when the file is not of that form (plain gzip: one stream, read_gz's serial path) or anything about it is inconsistent.
bool read_bgzf(const char *path, c2b_bytes &buf)
{
    int fd = open(path, O_RDONLY);
    if (fd < 0) return false;
    struct stat st;
    if (fstat(fd, &st) != 0 || st.st_size < 28) { close(fd); return false; }
    const size_t n = (size_t)st.st_size;
    void *mp = mmap(nullptr, n, PROT_READ, MAP_PRIVATE, fd, 0);
    close(fd);
    if (mp == MAP_FAILED) return false;
    const uint8_t *d = (const uint8_t *)mp;
    struct Member { size_t data, clen, out; uint32_t isize, crc; };
    std::vector<Member> mem;
    size_t p = 0, total = 0;
    bool ok = true;
    while (p < n) {
        if (n - p < 18 || d[p] != 0x1f || d[p + 1] != 0x8b || d[p + 2] != 8 || d[p + 3] != 4) { ok = false; break; }    // FLG = FEXTRA only
        const size_t xlen = d[p + 10] | ((size_t)d[p + 11] << 8);
        if (p + 12 + xlen > n) { ok = false; break; }
        size_t bsize = 0, q = p + 12;
        const size_t xe = q + xlen;
        while (q + 4 <= xe) {
            const size_t slen = d[q + 2] | ((size_t)d[q + 3] << 8);
            if (d[q] == 'B' && d[q + 1] == 'C' && slen == 2 && q + 6 <= xe) bsize = (d[q + 4] | ((size_t)d[q + 5] << 8)) + 1;
            q += 4 + slen;
        }
        if (bsize < 12 + xlen + 8 || p + bsize > n) { ok = false; break; }
        Member m;
        m.data = p + 12 + xlen;
        m.clen = bsize - (12 + xlen) - 8;
        const uint8_t *tr = d + p + bsize - 8;
        m.crc = tr[0] | ((uint32_t)tr[1] << 8) | ((uint32_t)tr[2] << 16) | ((uint32_t)tr[3] << 24);
        m.isize = tr[4] | ((uint32_t)tr[5] << 8) | ((uint32_t)tr[6] << 16) | ((uint32_t)tr[7] << 24);
        m.out = total;
        total += m.isize;
        mem.push_back(m);
        p += bsize;
    }
    if (!ok || mem.empty()) { munmap(mp, n); return false; }
    c2b_bytes out(total);
    int T = (int)std::thread::hardware_concurrency();
    T = std::max(1, std::min(T, 64));
    if (mem.size() < 64) T = 1;
    std::atomic<size_t> next(0);
    std::atomic<bool> bad(false);
    auto work = [&]() {
        z_stream zs;
        memset(&zs, 0, sizeof(zs));
        if (inflateInit2(&zs, -15) != Z_OK) { bad.store(true); return; }
        for (;;) {
            const size_t k0 = next.fetch_add(16);
            if (k0 >= mem.size() || bad.load()) break;
            for (size_t k = k0; k < std::min(mem.size(), k0 + 16); k++) {
                const Member &m = mem[k];
                if (m.isize == 0 && m.clen <= 2) continue;                  // the empty end-of-file block
                inflateReset(&zs);
                zs.next_in = (Bytef *)(d + m.data); zs.avail_in = (uInt)m.clen;
                zs.next_out = out.data() + m.out; zs.avail_out = m.isize;
                const int rc = inflate(&zs, Z_FINISH);
                if (rc != Z_STREAM_END || zs.avail_out != 0 || crc32(0L, out.data() + m.out, m.isize) != m.crc) { bad.store(true); break; }
            }
        }
        inflateEnd(&zs);
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(work);
    work();
    for (auto &x : th) x.join();
    munmap(mp, n);
    if (bad.load()) return false;
    buf.swap(out);
    return true;
}

bool read_gz(const char *path, c2b_bytes &buf, std::string &err)
{
    if (read_bgzf(path, buf)) return true;
    gzFile g = gzopen(path, "rb");
    if (!g) { err = std::string("cannot open ") + path; return false; }
    gzbuffer(g, 1 << 20);
    size_t used = 0;
    buf.resize(64 << 20);
    for (;;) {
        if (buf.size() - used < (16u << 20)) buf.resize(buf.size() * 2);
        int n = gzread(g, buf.data() + used, (unsigned)std::min<size_t>(buf.size() - used, 1u << 30));
        if (n < 0) { int e; err = gzerror(g, &e); gzclose(g); return false; }
        if (n == 0) break;
        used += (size_t)n;
    }
    gzclose(g);
    buf.resize(used);
    return true;
}

// (3) sharded exact dedup in file order and (4) the unique reads in first-seen order, from every record's sequence and hash:
// shared by the FASTQ front end and the SAM one (c2b_sam_dedup_buffer)
void dedup_records(const std::vector<Seq> &seq, const std::vector<uint64_t> &hv, int64_t n_rec, int T, c2b_fastq *F,
                   const std::function<void(const char *)> &lap)
{
    // (3) sharded exact dedup in file order
    struct Ent { int64_t first; int32_t count; };
    std::vector<std::vector<Ent>> found(T);
    auto shard = [&](int s) {
        size_t mine = 0;
        for (int64_t r = 0; r < n_rec; r++) mine += ((hv[(size_t)r] >> 40) % (uint64_t)T) == (uint64_t)s;
        size_t cap = 64;
        while (cap < mine * 2 + 8) cap <<= 1;
        std::vector<int32_t> slot(cap, -1);                // index into found[s]
        auto &E = found[s];
        for (int64_t r = 0; r < n_rec; r++) {
            const uint64_t h = hv[(size_t)r];
            if (((h >> 40) % (uint64_t)T) != (uint64_t)s) continue;
            size_t k = (size_t)h & (cap - 1);
            for (;;) {
                const int32_t e = slot[k];
                if (e < 0) { slot[k] = (int32_t)E.size(); E.push_back({r, 1}); break; }
                const Seq &a = seq[(size_t)E[(size_t)e].first], &b = seq[(size_t)r];
                if (hv[(size_t)E[(size_t)e].first] == h && a.len == b.len && memcmp(a.p, b.p, a.len) == 0) { E[(size_t)e].count++; break; }
                k = (k + 1) & (cap - 1);
            }
        }
    };
    {
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(shard, t);
        shard(0);
        for (auto &x : th) x.join();
    }

    lap("dedup");
    // (4) unique reads in first-seen order: the shards' entries are scattered to their first record (disjoint records, so
    // in parallel), a prefix count over the records numbers them -- no sort, no serial pass over the unique reads
    std::vector<int32_t> cnt_at((size_t)n_rec, 0);
    {
        auto scatter = [&](int t) { for (const Ent &e : found[(size_t)t]) cnt_at[(size_t)e.first] = e.count; };
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(scatter, t);
        scatter(0);
        for (auto &x : th) x.join();
    }
    std::vector<size_t> u0((size_t)T + 1, 0);              // unique reads / bytes before thread t's record range
    std::vector<int64_t> b0((size_t)T + 1, 0);
    std::vector<int32_t> mx((size_t)T, 0);
    auto rec_lo = [&](int t) { return n_rec * t / T; };
    {
        auto count = [&](int t) {
            size_t u = 0; int64_t by = 0; int32_t m = 0;
            for (int64_t r = rec_lo(t); r < rec_lo(t + 1); r++) if (cnt_at[(size_t)r]) { u++; by += seq[(size_t)r].len; m = std::max<int32_t>(m, (int32_t)seq[(size_t)r].len); }
            u0[(size_t)t + 1] = u; b0[(size_t)t + 1] = by; mx[(size_t)t] = m;
        };
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(count, t);
        count(0);
        for (auto &x : th) x.join();
    }
    for (int t = 0; t < T; t++) { u0[(size_t)t + 1] += u0[(size_t)t]; b0[(size_t)t + 1] += b0[(size_t)t]; F->max_len = std::max(F->max_len, mx[(size_t)t]); }
    const size_t nu = u0[(size_t)T];
    const int64_t tot = b0[(size_t)T];
    F->offsets.resize(nu + 1);
    F->counts.resize(nu);
    F->first_index.resize(nu);
    F->offsets[nu] = tot;
    F->seqs.reset(new uint8_t[(size_t)tot + 16]);
    {
        auto emit = [&](int t) {
            size_t u = u0[(size_t)t]; int64_t by = b0[(size_t)t];
            for (int64_t r = rec_lo(t); r < rec_lo(t + 1); r++) {
                const int32_t c = cnt_at[(size_t)r];
                if (!c) continue;
                const Seq &q = seq[(size_t)r];
                F->offsets[u] = by; F->counts[u] = c; F->first_index[u] = r;
                memcpy(F->seqs.get() + by, q.p, q.len);
                by += q.len; u++;
            }
        };
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(emit, t);
        emit(0);
        for (auto &x : th) x.join();
    }
    lap("emit");
}

}  // namespace

static std::string g_fastq_err;

bool c2b_fastq_read_gz(const char *path, c2b_bytes &buf, std::string &err) { return read_gz(path, buf, err); }
void c2b_fastq_set_error(const std::string &m) { g_fastq_err = m; }
int c2b_sam_line_error(int64_t line, int kind)
{
    g_fastq_err = "SAM text line " + std::to_string(line + 1) + (kind ? ": fewer than 10 tab-separated fields" : ": non-ASCII byte (out of contract)");
    return kind ? C2B_E_LIMIT : C2B_E_ARG;
}

extern "C" {

const char *c2b_fastq_last_error(void) { return g_fastq_err.c_str(); }

int c2b_fastq_dedup_buffer(const uint8_t *data, size_t n, int32_t n_threads, c2b_fastq **out)
{
    if (!out || (n && !data)) return C2B_E_ARG;
    c2b_fastq *F = new c2b_fastq();
    const bool verbose = getenv("C2B_FASTQ_VERBOSE") != nullptr;
    auto t_last = std::chrono::steady_clock::now();
    auto lap = [&](const char *what) {
        if (!verbose) return;
        auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[c2b_fastq] %-10s %.3f s\n", what, std::chrono::duration<double>(now - t_last).count());
        t_last = now;
    };
    int T = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
    T = std::max(1, std::min(T, 64));
    if (n < (1u << 20)) T = 1;

    // (1) line starts.  Thread t scans [cut[t], cut[t+1]); cuts sit just after a line terminator.
    std::vector<size_t> cut(T + 1, 0);
    cut[T] = n;
    for (int t = 1; t < T; t++) {
        size_t p = std::max(cut[t - 1], n / T * t);
        while (p < n && data[p] != '\n' && data[p] != '\r') p++;
        if (p < n) p += (data[p] == '\r' && p + 1 < n && data[p + 1] == '\n') ? 2 : 1;
        cut[t] = std::min(p, n);
    }
    std::vector<std::vector<uint64_t>> starts(T);          // per thread: line start offsets and content lengths
    std::vector<std::vector<uint32_t>> lens(T);
    auto scan = [&](int t) {
        size_t p = cut[t];
        const size_t e = cut[t + 1];
        auto &S = starts[t]; auto &L = lens[t];
        S.reserve((e - p) / 60 + 16); L.reserve((e - p) / 60 + 16);
        while (p < e) {
            const uint8_t *q = data + p;
            const uint8_t *nl = (const uint8_t *)memchr(q, '\n', e - p);
            const size_t a = nl ? (size_t)(nl - data) : e;
            const uint8_t *cr = (const uint8_t *)memchr(q, '\r', a - p);     // first CR before that LF
            if (cr) {                                                         // "\r\n" pair, or a lone '\r' (universal newlines)
                const size_t b = (size_t)(cr - data);
                S.push_back(p); L.push_back((uint32_t)(b - p));
                p = (nl && b + 1 == a) ? a + 1 : b + 1;
            } else {
                S.push_back(p); L.push_back((uint32_t)(a - p));
                p = nl ? a + 1 : e;
            }
        }
    };
    {
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(scan, t);
        scan(0);
        for (auto &x : th) x.join();
    }
    lap("lines");
    std::vector<size_t> line_base(T + 1, 0);
    for (int t = 0; t < T; t++) line_base[t + 1] = line_base[t] + starts[t].size();
    const size_t n_lines = line_base[T];
    const int64_t n_rec = (int64_t)((n_lines + 3) / 4);
    F->n_reads = n_rec;
    auto line_at = [&](size_t k, Seq &s) {
        int t = (int)(std::upper_bound(line_base.begin(), line_base.end(), k) - line_base.begin()) - 1;
        const size_t j = k - line_base[t];
        s.p = data + starts[t][j]; s.len = lens[t][j];
    };

    // (2) sequences (line 2 of every record, stripped) and their hashes
    std::vector<Seq> seq((size_t)n_rec);
    std::vector<uint64_t> hv((size_t)n_rec);
    auto hash_range = [&](int t) {
        const int64_t a = n_rec * t / T, b = n_rec * (t + 1) / T;
        for (int64_t r = a; r < b; r++) {
            Seq s; s.p = data; s.len = 0;
            const size_t k = (size_t)r * 4 + 1;
            if (k < n_lines) {
                line_at(k, s);
                while (s.len && is_space(s.p[0])) { s.p++; s.len--; }
                while (s.len && is_space(s.p[s.len - 1])) s.len--;
            }
            seq[(size_t)r] = s;
            hv[(size_t)r] = hash_bytes(s.p, s.len);
        }
    };
    {
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(hash_range, t);
        hash_range(0);
        for (auto &x : th) x.join();
    }

    lap("hash");
    dedup_records(seq, hv, n_rec, T, F, lap);
    *out = F;
    return C2B_OK;
}

int c2b_fastq_dedup(const char *path, int32_t n_threads, c2b_fastq **out)
{
    if (!path || !out) return C2B_E_ARG;
    c2b_bytes buf;
    std::string err;
    const size_t L = strlen(path);
    const bool gz = L > 3 && strcmp(path + L - 3, ".gz") == 0;            // CRISPRessoCORE.py:1820
    auto t0 = std::chrono::steady_clock::now();
    if (!gz) {                                             // plain file: map it, no copy
        int fd = open(path, O_RDONLY);
        if (fd < 0) { g_fastq_err = std::string("c2b_fastq_dedup: cannot open ") + path; return C2B_E_ARG; }
        struct stat st;
        if (fstat(fd, &st) == 0 && st.st_size > 0) {
            void *m = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
            if (m != MAP_FAILED) {
                madvise(m, (size_t)st.st_size, MADV_SEQUENTIAL);
                const int rc = c2b_fastq_dedup_buffer((const uint8_t *)m, (size_t)st.st_size, n_threads, out);
                munmap(m, (size_t)st.st_size);
                close(fd);
                return rc;
            }
        }
        close(fd);
    }
    if (!(gz ? read_gz(path, buf, err) : read_plain(path, buf, err))) { g_fastq_err = "c2b_fastq_dedup: " + err; return C2B_E_ARG; }
    if (getenv("C2B_FASTQ_VERBOSE"))
        fprintf(stderr, "[c2b_fastq] read       %.3f s (%zu bytes)\n", std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(), buf.size());
    return c2b_fastq_dedup_buffer(buf.data(), buf.size(), n_threads, out);
}

#ifdef C2B_EMU
// the CPU warp-emulator build (test infrastructure) has no device front end
int c2b_fastq_gpu_available(void) { return 0; }
int c2b_fastq_dedup_gpu(const char *, int32_t, c2b_fastq **out) { if (out) *out = nullptr; g_fastq_err = "c2b_fastq_dedup_gpu: not built (emulator)"; return C2B_E_STATE; }
int c2b_fastq_dedup_gpu_buffer(const uint8_t *, size_t, int32_t, c2b_fastq **out) { if (out) *out = nullptr; g_fastq_err = "c2b_fastq_dedup_gpu: not built (emulator)"; return C2B_E_STATE; }
int c2b_sam_dedup_gpu_buffer(const uint8_t *, size_t, int32_t, c2b_fastq **out) { if (out) *out = nullptr; g_fastq_err = "c2b_sam_dedup_gpu_buffer: not built (emulator)"; return C2B_E_STATE; }
#endif

int64_t c2b_fastq_n_reads(const c2b_fastq *f) { return f ? f->n_reads : 0; }
int64_t c2b_fastq_n_unique(const c2b_fastq *f) { return f ? (int64_t)f->counts.size() : 0; }
int32_t c2b_fastq_max_len(const c2b_fastq *f) { return f ? f->max_len : 0; }
const uint8_t *c2b_fastq_seqs(const c2b_fastq *f) { return f ? f->seqs.get() : nullptr; }
const int64_t *c2b_fastq_offsets(const c2b_fastq *f) { return f ? f->offsets.data() : nullptr; }
const int32_t *c2b_fastq_counts(const c2b_fastq *f) { return f ? f->counts.data() : nullptr; }
const int64_t *c2b_fastq_first_index(const c2b_fastq *f) { return f ? f->first_index.data() : nullptr; }
void c2b_fastq_free(c2b_fastq *f) { delete f; }

}  // extern "C"

// ------------------------------------------------------------------------------------------------ quality filter
// Replaces: filterFastqs.filterFastqs for single-end input (reference: CRISPResso2/filterFastqs.py:29-229, called at
// CRISPRessoCORE.py:3716-3717).  Binary-mode semantics of the reference: lines end at '\n' only, every line is
// rstrip()ped of ASCII whitespace, processing stops at the first record whose id line is empty; quality = byte - 33 in
// uint8 arithmetic (wraps below 33); a record is kept iff min(q) >= min_bp_qual_in_read (when set) and
// mean(q) >= min_av_read_qual (when set; exact integer test sum >= thr * n); with min_bp_qual_or_N set, bases with
// q < thr become 'N'.  Output: id, sequence, plus line, quality, each followed by '\n'; a ".gz" output is written as
// one gzip member per worker thread (a valid multi-member gzip file).
namespace {

inline bool is_bspace(uint8_t c) { return c == ' ' || (c >= 9 && c <= 13); }     // bytes.rstrip()

struct Line { const uint8_t *p; uint32_t len; };
typedef std::vector<Line, c2b_noinit_alloc<Line>> Lines;

// lines of a buffer (split at '\n' only, right-stripped like bytes.rstrip()), indexed by all host threads: thread t takes the
// lines that START in its byte range (ranges are cut right after a '\n'), then the pieces are laid end to end
void split_lines(const uint8_t *data, size_t n, Lines &lines)
{
    const int T = host_threads(n);
    std::vector<size_t> cut((size_t)T + 1, 0);
    cut[(size_t)T] = n;
    for (int t = 1; t < T; t++) {
        size_t p = std::max(cut[(size_t)t - 1], n / (size_t)T * (size_t)t);
        const uint8_t *nl = p < n ? (const uint8_t *)memchr(data + p, '\n', n - p) : nullptr;
        cut[(size_t)t] = nl ? (size_t)(nl - data) + 1 : n;
    }
    std::vector<Lines> part((size_t)T);
    run_threads(T, [&](int t) {
        Lines &L = part[(size_t)t];
        const size_t e0 = cut[(size_t)t + 1];
        L.reserve((e0 - cut[(size_t)t]) / 60 + 16);
        for (size_t p = cut[(size_t)t]; p < e0;) {
            const uint8_t *nl = (const uint8_t *)memchr(data + p, '\n', e0 - p);
            const size_t e = nl ? (size_t)(nl - data) : e0;
            size_t q = e;
            while (q > p && is_bspace(data[q - 1])) q--;
            L.push_back({data + p, (uint32_t)(q - p)});
            p = nl ? e + 1 : e0;
        }
    });
    if (T == 1) { lines.swap(part[0]); return; }
    std::vector<size_t> at((size_t)T + 1, 0);
    for (int t = 0; t < T; t++) at[(size_t)t + 1] = at[(size_t)t] + part[(size_t)t].size();
    lines.resize(at[(size_t)T]);
    run_threads(T, [&](int t) { if (!part[(size_t)t].empty()) memcpy(lines.data() + at[(size_t)t], part[(size_t)t].data(), part[(size_t)t].size() * sizeof(Line)); });
}

bool gz_member(const std::string &in, std::string &out)
{
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (deflateInit2(&zs, 6, Z_DEFLATED, 15 + 16, 8, Z_DEFAULT_STRATEGY) != Z_OK) return false;
    out.resize(deflateBound(&zs, (uLong)in.size()) + 64);
    zs.next_in = (Bytef *)in.data(); zs.avail_in = (uInt)in.size();
    zs.next_out = (Bytef *)&out[0]; zs.avail_out = (uInt)out.size();
    const int rc = deflate(&zs, Z_FINISH);
    const size_t n = zs.total_out;
    deflateEnd(&zs);
    if (rc != Z_STREAM_END) return false;
    out.resize(n);
    return true;
}

}  // namespace

extern "C" int c2b_fastq_filter(const char *path_in, const char *path_out, int32_t min_bp_qual_in_read, int32_t min_av_read_qual,
                                int32_t min_bp_qual_or_N, int32_t n_threads, int64_t *n_in, int64_t *n_out)
{
    if (!path_in || !path_out) return C2B_E_ARG;
    c2b_bytes buf;
    std::string err;
    const size_t Li = strlen(path_in), Lo = strlen(path_out);
    const bool gz_in = Li > 3 && strcmp(path_in + Li - 3, ".gz") == 0, gz_out = Lo > 3 && strcmp(path_out + Lo - 3, ".gz") == 0;
    if (!(gz_in ? read_gz(path_in, buf, err) : read_plain(path_in, buf, err))) { g_fastq_err = "c2b_fastq_filter: " + err; return C2B_E_ARG; }
    const uint8_t *data = buf.data();
    const size_t n = buf.size();
    Lines lines;
    split_lines(data, n, lines);
    // records up to the first empty id line
    int64_t n_rec = 0;
    while ((size_t)(4 * n_rec) < lines.size() && lines[(size_t)(4 * n_rec)].len > 0) n_rec++;
    auto line_or_empty = [&](size_t k) -> Line { return k < lines.size() ? lines[k] : Line{data, 0}; };
    int T = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
    T = std::max(1, std::min(T, 64));
    if (n_rec < 4096) T = 1;
    std::vector<std::string> outs(T);
    std::vector<int64_t> kept(T, 0);
    std::vector<int> fail_code(T, 0);
    auto work = [&](int t) {
        const int64_t a = n_rec * t / T, b = n_rec * (t + 1) / T;
        std::string &o = outs[t];
        o.reserve((size_t)(b - a) * 560);
        std::string masked;
        for (int64_t r = a; r < b; r++) {
            const Line id = lines[(size_t)(4 * r)], sq = line_or_empty((size_t)(4 * r + 1)), pl = line_or_empty((size_t)(4 * r + 2)),
                       ql = line_or_empty((size_t)(4 * r + 3));
            if (min_bp_qual_in_read) {
                if (ql.len == 0) { fail_code[t] = 1; return; }            // numpy.min of an empty array raises in the reference
                uint8_t mn = 255;
                for (uint32_t k = 0; k < ql.len; k++) mn = std::min<uint8_t>(mn, (uint8_t)(ql.p[k] - 33));
                if ((int)mn < min_bp_qual_in_read) continue;
            }
            if (min_av_read_qual) {
                if (ql.len == 0) continue;                                 // mean of nothing is nan: the comparison fails
                uint64_t sum = 0;
                for (uint32_t k = 0; k < ql.len; k++) sum += (uint8_t)(ql.p[k] - 33);
                if ((int64_t)sum < (int64_t)min_av_read_qual * (int64_t)ql.len) continue;
            }
            o.append((const char *)id.p, id.len); o.push_back('\n');
            if (min_bp_qual_or_N) {
                if (sq.len != ql.len) { fail_code[t] = 2; return; }       // boolean index of another length: IndexError in the reference
                masked.assign((const char *)sq.p, sq.len);
                for (uint32_t k = 0; k < ql.len; k++) if ((int)(uint8_t)(ql.p[k] - 33) < min_bp_qual_or_N) masked[k] = 'N';
                o.append(masked);
            } else o.append((const char *)sq.p, sq.len);
            o.push_back('\n');
            o.append((const char *)pl.p, pl.len); o.push_back('\n');
            o.append((const char *)ql.p, ql.len); o.push_back('\n');
            kept[t]++;
        }
        if (gz_out) { std::string z; if (!gz_member(o, z)) { fail_code[t] = 3; return; } o.swap(z); }
    };
    {
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(work, t);
        work(0);
        for (auto &x : th) x.join();
    }
    for (int t = 0; t < T; t++) if (fail_code[t]) {
        g_fastq_err = fail_code[t] == 1 ? "c2b_fastq_filter: empty quality line" : fail_code[t] == 2 ? "c2b_fastq_filter: sequence and quality lengths differ" : "c2b_fastq_filter: deflate failed";
        return fail_code[t] == 3 ? C2B_E_STATE : (fail_code[t] == 1 ? C2B_E_LIMIT : C2B_E_ARG);
    }
    int64_t tot = 0;
    for (int t = 0; t < T; t++) tot += kept[t];
    std::string tail;
    if (gz_out && n_rec == 0) { std::string e2; gz_member(e2, tail); }                  // an empty but valid gzip file
    if (!write_parts(path_out, outs, tail)) { g_fastq_err = std::string("c2b_fastq_filter: cannot write ") + path_out; return C2B_E_ARG; }
    if (n_in) *n_in = n_rec;
    if (n_out) *n_out = tot;
    return C2B_OK;
}


// Paired input of filterFastqs (reference: CRISPResso2/filterFastqs.py:230-407, the seven run_*_pair variants): the two files
// are read in lockstep, four lines each per record, until read 1's id line is empty; a pair is kept iff BOTH mates pass.
// Kept quirks: with only the min filter, or only the mean filter, mate 2 must be STRICTLY above the threshold (:262, :284:
// `min2 > min_bp_qual_in_read`, `mean2 > min_av_read_qual`); with min + mean but no masking the mean is tested first (:300),
// so an empty quality line drops the pair (mean of nothing is nan) instead of raising; every other order tests the min
// first, where numpy.min of an empty array raises (-> C2B_E_LIMIT here).
namespace {

bool load_lines(const char *path, c2b_bytes &buf, Lines &lines, std::string &err)
{
    const size_t Lp = strlen(path);
    const bool gz = Lp > 3 && strcmp(path + Lp - 3, ".gz") == 0;
    if (!(gz ? read_gz(path, buf, err) : read_plain(path, buf, err))) return false;
    split_lines(buf.data(), buf.size(), lines);
    return true;
}

}  // namespace

extern "C" int c2b_fastq_filter_pair(const char *path1_in, const char *path2_in, const char *path1_out, const char *path2_out,
                                     int32_t min_bp_qual_in_read, int32_t min_av_read_qual, int32_t min_bp_qual_or_N,
                                     int32_t n_threads, int64_t *n_in, int64_t *n_out)
{
    if (!path1_in || !path2_in || !path1_out || !path2_out) return C2B_E_ARG;
    c2b_bytes buf1, buf2;
    Lines l1, l2;
    std::string err;
    if (!load_lines(path1_in, buf1, l1, err) || !load_lines(path2_in, buf2, l2, err)) { g_fastq_err = "c2b_fastq_filter_pair: " + err; return C2B_E_ARG; }
    static const uint8_t nothing = 0;
    auto at = [&](const Lines &L, size_t k) -> Line { return k < L.size() ? L[k] : Line{&nothing, 0}; };
    int64_t n_rec = 0;
    while ((size_t)(4 * n_rec) < l1.size() && l1[(size_t)(4 * n_rec)].len > 0) n_rec++;
    const bool bp = min_bp_qual_in_read != 0, rq = min_av_read_qual != 0, bpn = min_bp_qual_or_N != 0;
    const bool strict2 = (bp != rq) && !bpn;                 // run_mBP_pair / run_mRQ_pair: mate 2 strictly above
    const bool mean_first = bp && rq && !bpn;                // run_mBP_mRQ_pair
    const size_t o1 = strlen(path1_out), o2 = strlen(path2_out);
    const bool gz1 = o1 > 3 && strcmp(path1_out + o1 - 3, ".gz") == 0, gz2 = o2 > 3 && strcmp(path2_out + o2 - 3, ".gz") == 0;
    int T = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
    T = std::max(1, std::min(T, 64));
    if (n_rec < 4096) T = 1;
    std::vector<std::string> outs1(T), outs2(T);
    std::vector<int64_t> kept(T, 0);
    std::vector<int> fail_code(T, 0);
    auto qmin = [](const Line &q) { uint8_t mn = 255; for (uint32_t k = 0; k < q.len; k++) mn = std::min<uint8_t>(mn, (uint8_t)(q.p[k] - 33)); return (int)mn; };
    auto qsum = [](const Line &q) { uint64_t sm = 0; for (uint32_t k = 0; k < q.len; k++) sm += (uint8_t)(q.p[k] - 33); return (int64_t)sm; };
    auto work = [&](int t) {
        const int64_t a = n_rec * t / T, b = n_rec * (t + 1) / T;
        std::string &w1 = outs1[t], &w2 = outs2[t];
        w1.reserve((size_t)(b - a) * 560); w2.reserve((size_t)(b - a) * 560);
        std::string masked;
        auto emit = [&](std::string &o, const Line &id, const Line &sq, const Line &pl, const Line &ql) -> bool {
            o.append((const char *)id.p, id.len); o.push_back('\n');
            if (bpn) {
                if (sq.len != ql.len) return false;          // boolean index of another length: IndexError in the reference
                masked.assign((const char *)sq.p, sq.len);
                for (uint32_t k = 0; k < ql.len; k++) if ((int)(uint8_t)(ql.p[k] - 33) < min_bp_qual_or_N) masked[k] = 'N';
                o.append(masked);
            } else o.append((const char *)sq.p, sq.len);
            o.push_back('\n');
            o.append((const char *)pl.p, pl.len); o.push_back('\n');
            o.append((const char *)ql.p, ql.len); o.push_back('\n');
            return true;
        };
        for (int64_t r = a; r < b; r++) {
            const size_t k = (size_t)(4 * r);
            const Line id1 = l1[k], sq1 = at(l1, k + 1), pl1 = at(l1, k + 2), ql1 = at(l1, k + 3);
            const Line id2 = at(l2, k), sq2 = at(l2, k + 1), pl2 = at(l2, k + 2), ql2 = at(l2, k + 3);
            auto mean_ok = [&]() {
                if (ql1.len == 0 || ql2.len == 0) return false;                        // nan compares false
                const int64_t t1 = (int64_t)min_av_read_qual * ql1.len, t2 = (int64_t)min_av_read_qual * ql2.len;
                return qsum(ql1) >= t1 && (strict2 ? qsum(ql2) > t2 : qsum(ql2) >= t2);
            };
            auto min_ok = [&](bool &raised) {
                if (ql1.len == 0 || ql2.len == 0) { raised = true; return false; }       // numpy.min of an empty array raises
                return qmin(ql1) >= min_bp_qual_in_read && (strict2 ? qmin(ql2) > min_bp_qual_in_read : qmin(ql2) >= min_bp_qual_in_read);
            };
            bool raised = false, keep = true;
            if (mean_first) keep = mean_ok() && min_ok(raised);
            else {
                if (bp) keep = min_ok(raised);
                if (keep && rq) keep = mean_ok();
            }
            if (raised) { fail_code[t] = 1; return; }
            if (!keep) continue;
            if (!emit(w1, id1, sq1, pl1, ql1) || !emit(w2, id2, sq2, pl2, ql2)) { fail_code[t] = 2; return; }
            kept[t]++;
        }
        if (gz1) { std::string z; if (!gz_member(w1, z)) { fail_code[t] = 3; return; } w1.swap(z); }
        if (gz2) { std::string z; if (!gz_member(w2, z)) { fail_code[t] = 3; return; } w2.swap(z); }
    };
    {
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(work, t);
        work(0);
        for (auto &x : th) x.join();
    }
    for (int t = 0; t < T; t++) if (fail_code[t]) {
        g_fastq_err = fail_code[t] == 1 ? "c2b_fastq_filter_pair: empty quality line" : fail_code[t] == 2 ? "c2b_fastq_filter_pair: sequence and quality lengths differ" : "c2b_fastq_filter_pair: deflate failed";
        return fail_code[t] == 3 ? C2B_E_STATE : (fail_code[t] == 1 ? C2B_E_LIMIT : C2B_E_ARG);
    }
    int64_t tot = 0;
    for (int f = 0; f < 2; f++) {
        std::string tail;
        if ((f ? gz2 : gz1) && n_rec == 0) { std::string e2; gz_member(e2, tail); }
        if (!write_parts(f ? path2_out : path1_out, f ? outs2 : outs1, tail)) {
            g_fastq_err = std::string("c2b_fastq_filter_pair: cannot write ") + (f ? path2_out : path1_out);
            return C2B_E_ARG;
        }
    }
    for (int t = 0; t < T; t++) tot += kept[t];
    if (n_in) *n_in = n_rec;
    if (n_out) *n_out = tot;
    return C2B_OK;
}


// ------------------------------------------------------------------------------------------ reverse-complement merge
// replaces: the count transfer at the head of the quantification loop (CRISPRessoCORE.py:3964-3975): walking the unique
// reads in first-seen order, a read with a non-zero count absorbs the count of its reverse complement (CRISPRessoShared.py:
// 399-403: upper-cased, A<->T, C<->G, N, '_', '-' kept), whose count drops to 0; a palindromic read absorbs itself (its
// count doubles, as in the reference).  Reads holding any other symbol are left alone (the reference raises KeyError there).
// `member` (optional, one byte per read): only reads with member != 0 are in the cache (the aligned ones, :1983-1985).
// Hashing and the partner search run on host threads; the sweep that applies the rule is serial (it is order-dependent).
extern "C" int c2b_rc_merge_weights(const uint8_t *seqs, const int64_t *offsets, int64_t n, const int32_t *counts,
                                    const uint8_t *member, int32_t *weights, int32_t n_threads)
{
    if (!offsets || !counts || !weights || n < 0 || (n && !seqs)) return -2;
    int T = n_threads > 0 ? n_threads : (int)std::max(1u, std::thread::hardware_concurrency());
    T = (int)std::min<int64_t>(T, std::max<int64_t>(1, n / 4096));
    size_t cap = 16;
    while (cap < (size_t)n * 2 + 16) cap <<= 1;
    std::vector<int64_t> table(cap, -1), partner((size_t)n, -1);
    std::vector<uint64_t> hv((size_t)n);
    auto run = [&](const std::function<void(int64_t, int64_t)> &fn) {
        std::vector<std::thread> th;
        for (int t = 1; t < T; t++) th.emplace_back(fn, n * t / T, n * (t + 1) / T);
        fn(0, n / T);
        for (auto &x : th) x.join();
    };
    run([&](int64_t lo, int64_t hi) { for (int64_t k = lo; k < hi; k++) hv[(size_t)k] = hash_bytes(seqs + offsets[k], (size_t)(offsets[k + 1] - offsets[k])); });
    for (int64_t k = 0; k < n; k++) {                       // unique reads: every key is new
        if (member && !member[k]) continue;
        size_t h = (size_t)hv[(size_t)k] & (cap - 1);
        while (table[h] >= 0) h = (h + 1) & (cap - 1);
        table[h] = k;
    }
    static const struct Comp { uint8_t t[256]; Comp() { memset(t, 0, sizeof t); const char *a = "ACGTN_-acgtn", *b = "TGCAN_-TGCAN"; for (int i = 0; a[i]; i++) t[(uint8_t)a[i]] = (uint8_t)b[i]; } } comp;
    run([&](int64_t lo, int64_t hi) {
        std::vector<uint8_t> rc;
        for (int64_t k = lo; k < hi; k++) {
            if (member && !member[k]) continue;
            const uint8_t *p = seqs + offsets[k];
            const size_t L = (size_t)(offsets[k + 1] - offsets[k]);
            rc.resize(L);
            bool ok = true;
            for (size_t i = 0; i < L; i++) { const uint8_t c = comp.t[p[L - 1 - i]]; if (!c) { ok = false; break; } rc[i] = c; }
            if (!ok) continue;
            const uint64_t hh = hash_bytes(rc.data(), L);
            size_t h = (size_t)hh & (cap - 1);
            while (table[h] >= 0) {
                const int64_t j = table[h];
                if (hv[(size_t)j] == hh && (size_t)(offsets[j + 1] - offsets[j]) == L && memcmp(seqs + offsets[j], rc.data(), L) == 0) { partner[(size_t)k] = j; break; }
                h = (h + 1) & (cap - 1);
            }
        }
    });
    for (int64_t k = 0; k < n; k++) weights[k] = counts[k];
    for (int64_t k = 0; k < n; k++) {
        if (weights[k] == 0 || (member && !member[k])) continue;
        const int64_t j = partner[(size_t)k];
        if (j >= 0 && weights[j] > 0) { const int32_t tot = weights[k] + weights[j]; weights[j] = 0; weights[k] = tot; }
    }
    return 0;
}

// Reads outside the engine's contract (crispresso2_b200/core.py: screen_reads): empty, longer than max_len, or holding a
// symbol other than A C G T N.  out[k] = 1 for such reads.  Host threads.  -> number of flagged reads
extern "C" int64_t c2b_screen_reads(const uint8_t *seqs, const int64_t *offsets, int64_t n, int32_t max_len, uint8_t *out, int32_t n_threads)
{
    if (!offsets || !out || n < 0 || (n && !seqs)) return -2;
    int T = n_threads > 0 ? n_threads : (int)std::max(1u, std::thread::hardware_concurrency());
    T = (int)std::min<int64_t>(T, std::max<int64_t>(1, n / 8192));
    static const struct Ok { uint8_t t[256]; Ok() { memset(t, 0, sizeof t); for (const char *a = "ACGTN"; *a; a++) t[(uint8_t)*a] = 1; } } ok;
    std::vector<int64_t> bad((size_t)T, 0);
    auto work = [&](int t) {
        const int64_t lo = n * t / T, hi = n * (t + 1) / T;
        int64_t nb = 0;
        for (int64_t k = lo; k < hi; k++) {
            const int64_t L = offsets[k + 1] - offsets[k];
            uint8_t b = (L < 1 || L > max_len) ? 1 : 0;
            const uint8_t *p = seqs + offsets[k];
            uint8_t all = 1;
            for (int64_t i = 0; i < L; i++) all &= ok.t[p[i]];
            b |= (uint8_t)(all ^ 1);
            out[k] = b; nb += b;
        }
        bad[(size_t)t] = nb;
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(work, t);
    work(0);
    for (auto &x : th) x.join();
    int64_t tot = 0;
    for (int64_t v : bad) tot += v;
    return tot;
}

// aln_stats of the serial process_fastq branch (CRISPRessoCORE.py:1956-1999) from a batch's per-read records, one threaded
// pass: out[0..10] = N_TOT_READS, N_CACHED_ALN, N_CACHED_NOTALN, N_COMPUTED_ALN, N_COMPUTED_NOTALN, N_GLOBAL_SUBS,
// N_SUBS_OUTSIDE_WINDOW, N_MODS_IN_WINDOW, N_MODS_OUTSIDE_WINDOW, N_READS_IRREGULAR_ENDS, READ_LENGTH (the first aligned
// read's alignment length, :1980).  The statistics of an aligned unique read are those of its best_match_name (best_ref, the
// LAST winner).  aligned[k] = 1 for reads with best_match_score > 0.  The host side uses this as the cross-check of the
// kernel's own sums (core.py) -- the Python loop it replaces cost 0.11 s per million unique reads.
extern "C" int c2b_serial_stats(const c2b_read_rec *recs, const c2b_aln_rec *alns, const int32_t *counts, int64_t n, int32_t nr,
                                int64_t *out, uint8_t *aligned, int32_t n_threads)
{
    if (n < 0 || nr < 1 || !out || (n && (!recs || !alns || !counts || !aligned))) return C2B_E_ARG;
    int T = n_threads > 0 ? n_threads : (int)std::max(1u, std::thread::hardware_concurrency());
    T = (int)std::min<int64_t>(std::min(T, 32), std::max<int64_t>(1, n / 65536));
    std::vector<std::vector<int64_t>> part((size_t)T, std::vector<int64_t>(12, 0));
    auto work = [&](int t) {
        std::vector<int64_t> &o = part[(size_t)t];
        o[11] = -1;                                            // index of this slice's first aligned read
        const int64_t lo = n * t / T, hi = n * (t + 1) / T;
        for (int64_t k = lo; k < hi; k++) {
            const int64_t c = counts[k];
            const bool al = recs[k].best_score_milli > 0;
            aligned[k] = al ? 1 : 0;
            o[0] += c;
            if (!al) { o[4]++; o[2] += c - 1; continue; }
            o[3]++; o[1] += c - 1;
            int col = nr > 1 ? recs[k].best_ref : 0;
            if (col < 0 || col >= nr) col = 0;
            const c2b_aln_rec &a = alns[k * nr + col];
            const int64_t in_win = (int64_t)a.substitution_n + a.deletion_n + a.insertion_n;
            const int64_t total = (int64_t)a.n_ins_all + a.n_del_pos_all + a.n_sub_all;
            o[5] += c * a.n_sub_all; o[6] += c * ((int64_t)a.n_sub_all - a.substitution_n);
            o[7] += c * in_win; o[8] += c * (total - in_win);
            if (a.irregular_ends) o[9] += c;
            if (o[11] < 0) { o[11] = k; o[10] = a.aln_len; }
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(work, t);
    work(0);
    for (auto &x : th) x.join();
    for (int j = 0; j < 11; j++) out[j] = 0;
    bool have_len = false;
    for (int t = 0; t < T; t++) {
        for (int j = 0; j < 10; j++) out[j] += part[(size_t)t][(size_t)j];
        if (!have_len && part[(size_t)t][11] >= 0) { out[10] = part[(size_t)t][10]; have_len = true; }
    }
    return C2B_OK;
}

// ------------------------------------------------------------------------------------------------ annotated output
// Replaces the record loops of process_fastq_write_out (CRISPRessoCORE.py:2293-2346) and process_single_fastq_write_bam_out
// (:2387-2502): the input FASTQ is read again, split into records by the text-mode readline() rules of the ingest (universal
// newlines; a record starts at every line and takes the next three, present or not), each record's sequence found in a hash of
// the unique reads (byte compare), and the record written with its read's annotation (c2b_annotation, built on the device).
namespace {

struct TLine { size_t p; uint32_t len; };

// lines under universal newlines ("\n", "\r\n", lone "\r"), indexed by all host threads from cuts placed right after a terminator
void split_text_lines(const uint8_t *data, size_t n, std::vector<TLine> &lines)
{
    const int T = host_threads(n);
    std::vector<size_t> cut((size_t)T + 1, 0);
    cut[(size_t)T] = n;
    for (int t = 1; t < T; t++) {
        size_t p = std::max(cut[(size_t)t - 1], n / (size_t)T * (size_t)t);
        while (p < n && data[p] != '\n' && data[p] != '\r') p++;
        if (p < n) p += (data[p] == '\r' && p + 1 < n && data[p + 1] == '\n') ? 2 : 1;
        cut[(size_t)t] = std::min(p, n);
    }
    std::vector<std::vector<TLine>> part((size_t)T);
    run_threads(T, [&](int t) {
        std::vector<TLine> &L = part[(size_t)t];
        size_t p = cut[(size_t)t];
        const size_t e = cut[(size_t)t + 1];
        L.reserve((e - p) / 60 + 16);
        while (p < e) {
            size_t q = p;
            while (q < e && data[q] != '\n' && data[q] != '\r') q++;
            L.push_back({p, (uint32_t)(q - p)});
            p = q < e ? q + ((data[q] == '\r' && q + 1 < e && data[q + 1] == '\n') ? 2 : 1) : e;
        }
    });
    size_t tot = 0;
    for (auto &L : part) tot += L.size();
    lines.clear();
    lines.reserve(tot);
    for (auto &L : part) lines.insert(lines.end(), L.begin(), L.end());
}

struct UniqueIndex {                                         // exact sequence -> unique read index
    const uint8_t *seqs; const int64_t *off; std::vector<int64_t> slot; uint64_t mask = 0;
    UniqueIndex(const uint8_t *s, const int64_t *o, int64_t n) : seqs(s), off(o)
    {
        size_t cap = 16;
        while (cap < (size_t)n * 2) cap <<= 1;
        slot.assign(cap, -1); mask = cap - 1;
        for (int64_t u = 0; u < n; u++) {
            uint64_t h = hash_bytes(s + o[u], (size_t)(o[u + 1] - o[u])) & mask;
            while (slot[h] >= 0) h = (h + 1) & mask;
            slot[h] = u;
        }
    }
    int64_t find(const uint8_t *p, size_t len) const
    {
        uint64_t h = hash_bytes(p, len) & mask;
        for (; slot[h] >= 0; h = (h + 1) & mask) {
            const int64_t u = slot[h];
            if ((size_t)(off[u + 1] - off[u]) == len && (len == 0 || memcmp(seqs + off[u], p, len) == 0)) return u;
        }
        return -1;
    }
};

struct TextInput {
    c2b_bytes buf;
    std::vector<TLine> lines;
    bool last_open = false;                                  // the last line has no terminator
    std::string err;
    bool load(const char *path)
    {
        const size_t L = strlen(path);
        const bool gz = L > 3 && strcmp(path + L - 3, ".gz") == 0;          // CRISPRessoCORE.py:2288, :2380
        if (!(gz ? read_gz(path, buf, err) : read_plain(path, buf, err))) return false;
        const size_t n = buf.size();
        std::atomic<bool> wide(false);
        const int T = host_threads(n);
        run_threads(T, [&](int t) {
            const size_t a = n * (size_t)t / T, b = n * (size_t)(t + 1) / T;
            for (size_t i = a; i < b; i++) if (buf[i] & 0x80) { wide.store(true); return; }
        });
        if (wide.load()) { err = "non-ASCII byte in the FASTQ input (out of contract for the annotated outputs)"; return false; }
        split_text_lines(buf.data(), n, lines);
        last_open = n && buf[n - 1] != '\n' && buf[n - 1] != '\r';
        return true;
    }
    bool has(size_t k) const { return k < lines.size(); }
    bool ends(size_t k) const { return k + 1 < lines.size() || !last_open; }
    Seq stripped(size_t k) const
    {
        Seq s{buf.data(), 0};
        if (!has(k)) return s;
        s.p = buf.data() + lines[k].p; s.len = lines[k].len;
        while (s.len && is_space(s.p[0])) { s.p++; s.len--; }
        while (s.len && is_space(s.p[s.len - 1])) s.len--;
        return s;
    }
};

}  // namespace

// FASTQ: id + seq + "\n" + plus + annotation + "\n" + qual per record (id and quality keep their newline), gzip, one member per
// thread and per 32 MB of text (a multi-member file whose decompressed bytes are what gzip.open(.., 'wt') would have written)
extern "C" int c2b_annotate_write_fastq(const c2b_annotation *a, const uint8_t *seqs, const int64_t *offsets, int64_t n_unique,
                                        const char *in_path, const char *out_path, int32_t n_threads)
{
    if (!a || !in_path || !out_path || n_unique != a->n || (n_unique && !offsets)) { g_fastq_err = "c2b_annotate_write_fastq: bad argument"; return C2B_E_ARG; }
    TextInput in;
    if (!in.load(in_path)) { g_fastq_err = "c2b_annotate_write_fastq: " + in.err; return C2B_E_ARG; }
    const UniqueIndex idx(seqs, offsets, n_unique);
    const int64_t n_rec = (int64_t)((in.lines.size() + 3) / 4);
    int T = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
    T = std::max(1, std::min(T, 64));
    if (n_rec < 4096) T = 1;
    std::vector<std::string> outs((size_t)T);
    std::vector<int> bad((size_t)T, 0);
    const uint8_t *D = in.buf.data();
    run_threads(T, [&](int t) {
        const int64_t lo = n_rec * t / T, hi = n_rec * (t + 1) / T;
        std::string o, z;
        o.reserve(40 << 20);
        auto flush = [&]() {
            if (!gz_member(o, z)) return false;
            outs[(size_t)t] += z; o.clear();
            return true;
        };
        for (int64_t r = lo; r < hi; r++) {
            const size_t k = (size_t)(4 * r);
            const Seq sq = in.stripped(k + 1), pl = in.stripped(k + 2);
            const int64_t u = idx.find(sq.p, sq.len);
            if (u < 0) { bad[(size_t)t] = 1; return; }
            o.append((const char *)D + in.lines[k].p, in.lines[k].len);
            if (in.ends(k)) o.push_back('\n');
            o.append((const char *)sq.p, sq.len); o.push_back('\n');
            o.append((const char *)pl.p, pl.len);
            o.append((const char *)a->ann.data() + a->ann_off[(size_t)u], (size_t)(a->ann_off[(size_t)u + 1] - a->ann_off[(size_t)u]));
            o.push_back('\n');
            if (in.has(k + 3)) { o.append((const char *)D + in.lines[k + 3].p, in.lines[k + 3].len); if (in.ends(k + 3)) o.push_back('\n'); }
            if (o.size() >= (32u << 20) && !flush()) { bad[(size_t)t] = 2; return; }
        }
        if (!o.empty() && !flush()) bad[(size_t)t] = 2;
    });
    for (int b : bad) if (b) {
        g_fastq_err = b == 1 ? "c2b_annotate_write_fastq: a read sequence is in neither variantCache nor the not-aligned reads" : "c2b_annotate_write_fastq: deflate failed";
        return b == 1 ? C2B_E_ARG : C2B_E_STATE;
    }
    std::string tail;
    bool any = false;
    for (auto &s : outs) any |= !s.empty();
    if (!any) { std::string e2; gz_member(e2, tail); }                 // an empty but valid gzip file
    if (!write_parts(out_path, outs, tail)) { g_fastq_err = std::string("c2b_annotate_write_fastq: cannot write ") + out_path; return C2B_E_STATE; }
    return C2B_OK;
}

// SAM: the header, then one line per record until the first record whose stripped id line is at most one character (the loop
// condition of :2392); unaligned reads as flag 4, aligned ones at the first aligned reference's chr / start with its CIGAR, flag,
// MAPQ, and reverse-complemented sequence / reversed quality when that reference's aln_strand is '-' (:2462-2469).  Records the
// id and quality of each unique read's last record in the handle (sam_entry of :2497).
extern "C" int c2b_annotate_write_sam(c2b_annotation *a, const uint8_t *seqs, const int64_t *offsets, int64_t n_unique,
                                      const char *in_path, const char *sam_path, const char *header, int32_t n_names,
                                      const char *const *chr, const char *const *pos, const uint8_t *rev, int32_t n_threads)
{
    if (!a || !in_path || !sam_path || !header || n_unique != a->n || (n_unique && !offsets) || n_names < 0 ||
        (n_names && (!chr || !pos || !rev))) { g_fastq_err = "c2b_annotate_write_sam: bad argument"; return C2B_E_ARG; }
    TextInput in;
    if (!in.load(in_path)) { g_fastq_err = "c2b_annotate_write_sam: " + in.err; return C2B_E_ARG; }
    const UniqueIndex idx(seqs, offsets, n_unique);
    int64_t n_rec = 0;
    while (in.has((size_t)(4 * n_rec)) && in.stripped((size_t)(4 * n_rec)).len > 1) n_rec++;
    int T = n_threads > 0 ? n_threads : (int)std::thread::hardware_concurrency();
    T = std::max(1, std::min(T, 64));
    if (n_rec < 4096) T = 1;
    std::vector<std::string> outs((size_t)T + 1);
    outs[0] = header;
    std::vector<int64_t> rec_u((size_t)n_rec, -1);
    std::vector<int> bad((size_t)T, 0);
    unsigned char comp[256];
    for (int c = 0; c < 256; c++) comp[c] = 0;
    comp['A'] = 'T'; comp['C'] = 'G'; comp['G'] = 'C'; comp['T'] = 'A'; comp['N'] = 'N'; comp['_'] = '_'; comp['-'] = '-';
    run_threads(T, [&](int t) {
        const int64_t lo = n_rec * t / T, hi = n_rec * (t + 1) / T;
        std::string &o = outs[(size_t)t + 1];
        std::string s2, q2;
        for (int64_t r = lo; r < hi; r++) {
            const size_t k = (size_t)(4 * r);
            const Seq id = in.stripped(k), sq = in.stripped(k + 1), ql = in.stripped(k + 3);
            const int64_t u = idx.find(sq.p, sq.len);
            if (u < 0) { bad[(size_t)t] = 1; return; }
            rec_u[(size_t)r] = u;
            const uint8_t fl = a->flag[(size_t)u];
            const int f = a->first[(size_t)u];
            if (fl != 255 && (f < 0 || f >= n_names)) { bad[(size_t)t] = 2; return; }
            o.append((const char *)id.p + 1, id.len - 1);
            const char *sp = (const char *)sq.p, *qp = (const char *)ql.p;
            if (fl == 255) o += "\t4\t*\t0\t0\t*\t*\t0\t0\t";
            else {
                o.push_back('\t'); o += std::to_string((int)fl); o.push_back('\t'); o += chr[f]; o.push_back('\t'); o += pos[f];
                o.push_back('\t'); o += std::to_string(a->mapq[(size_t)u]); o.push_back('\t');
                o.append((const char *)a->cig.data() + a->cig_off[(size_t)u], (size_t)(a->cig_off[(size_t)u + 1] - a->cig_off[(size_t)u]));
                o += "\t*\t0\t0\t";
                if (rev[f]) {                                  // CRISPRessoShared.reverse_complement (:399-403), quality reversed
                    s2.assign(sq.len, ' '); q2.assign(ql.len, ' ');
                    for (uint32_t i = 0; i < sq.len; i++) {
                        unsigned char c = sq.p[sq.len - 1 - i];
                        if (c >= 'a' && c <= 'z') c = (unsigned char)(c - 32);
                        if (!comp[c]) { bad[(size_t)t] = 3; return; }
                        s2[i] = (char)comp[c];
                    }
                    for (uint32_t i = 0; i < ql.len; i++) q2[i] = (char)ql.p[ql.len - 1 - i];
                    sp = s2.data(); qp = q2.data();
                }
            }
            o.append(sp, sq.len); o.push_back('\t'); o.append(qp, ql.len);
            o += "\tc2:Z:";
            const int64_t a0 = a->ann_off[(size_t)u], a1 = a->ann_off[(size_t)u + 1];
            if (a1 > a0) o.append((const char *)a->ann.data() + a0 + 1, (size_t)(a1 - a0 - 1));
            o.push_back('\n');
        }
    });
    for (int b : bad) if (b) {
        g_fastq_err = b == 1 ? "c2b_annotate_write_sam: a read sequence is in neither variantCache nor the not-aligned reads"
                    : b == 2 ? "c2b_annotate_write_sam: reference name id out of range" : "c2b_annotate_write_sam: symbol without a complement";
        return C2B_E_ARG;
    }
    if (!write_parts(sam_path, outs, std::string())) { g_fastq_err = std::string("c2b_annotate_write_sam: cannot write ") + sam_path; return C2B_E_STATE; }
    a->last_rec.assign((size_t)n_unique, -1);
    for (int64_t r = 0; r < n_rec; r++) a->last_rec[(size_t)rec_u[(size_t)r]] = r;
    a->rec.clear();
    a->rec_off.assign(1, 0);
    a->rec_off.reserve((size_t)n_unique * 2 + 1);
    for (int64_t u = 0; u < n_unique; u++) {
        const int64_t r = a->last_rec[(size_t)u];
        if (r >= 0) {
            const Seq id = in.stripped((size_t)(4 * r)), ql = in.stripped((size_t)(4 * r + 3));
            a->rec.append((const char *)id.p + 1, id.len - 1); a->rec_off.push_back((int64_t)a->rec.size());
            a->rec.append((const char *)ql.p, ql.len);
        } else a->rec_off.push_back((int64_t)a->rec.size());
        a->rec_off.push_back((int64_t)a->rec.size());
    }
    return C2B_OK;
}

// ------------------------------------------------------------------------------------------------ SAM text (process_bam)
// Replaces the two `samtools view` loops of process_bam (CRISPRessoCORE.py:2047-2057 and :2251-2262), whose lines are read in
// text mode (universal newlines) and split as line.rstrip().split("\t"): the read is field 10.
namespace {

// field 10 of line.rstrip().split("\t"): [s0, s1) within the line, e = the rstrip end; false when there are fewer than 10 fields
bool sam_field10(const uint8_t *p, uint32_t len, uint32_t &s0, uint32_t &s1, uint32_t &e)
{
    e = len;
    while (e && is_space(p[e - 1])) e--;
    uint32_t i = 0;
    for (int tabs = 0; tabs < 9; tabs++) {
        const uint8_t *q = (const uint8_t *)memchr(p + i, '\t', e - i);
        if (!q) return false;
        i = (uint32_t)(q - p) + 1;
    }
    s0 = i;
    const uint8_t *q = (const uint8_t *)memchr(p + i, '\t', e - i);
    s1 = q ? (uint32_t)(q - p) : e;
    return true;
}

// the first bad line of lines [lo, hi) as (line << 1) | kind (kind 0: a non-ASCII byte, 1: fewer than 10 fields), or -1
int64_t sam_first_bad(const uint8_t *data, const std::vector<TLine> &lines, size_t lo, size_t hi)
{
    for (size_t k = lo; k < hi; k++) {
        const uint8_t *p = data + lines[k].p;
        for (uint32_t i = 0; i < lines[k].len; i++) if (p[i] & 0x80) return (int64_t)(k << 1);
        uint32_t s0, s1, e;
        if (!sam_field10(p, lines[k].len, s0, s1, e)) return (int64_t)((k << 1) | 1);
    }
    return -1;
}

int sam_threads(size_t n, int asked)
{
    int T = asked > 0 ? asked : (int)std::thread::hardware_concurrency();
    T = std::max(1, std::min(T, 64));
    return n < (1u << 20) ? 1 : T;
}

}  // namespace

// pass 1 on the host threads: the same c2b_fastq result as c2b_sam_dedup_gpu_buffer
extern "C" int c2b_sam_dedup_buffer(const uint8_t *data, size_t n, int32_t n_threads, c2b_fastq **out)
{
    if (!out || (n && !data)) return C2B_E_ARG;
    *out = nullptr;
    std::vector<TLine> lines;
    split_text_lines(data, n, lines);
    const int64_t n_rec = (int64_t)lines.size();
    if (n_rec >= (int64_t)INT32_MAX / 2) { g_fastq_err = "c2b_sam_dedup_buffer: more than 2^30 lines"; return C2B_E_LIMIT; }
    const int T = sam_threads(n, n_threads);
    std::vector<Seq> seq((size_t)n_rec);
    std::vector<uint64_t> hv((size_t)n_rec);
    std::vector<int64_t> bad((size_t)T, -1);
    run_threads(T, [&](int t) {
        const int64_t lo = n_rec * t / T, hi = n_rec * (t + 1) / T;
        bad[(size_t)t] = sam_first_bad(data, lines, (size_t)lo, (size_t)hi);
        if (bad[(size_t)t] >= 0) return;
        for (int64_t r = lo; r < hi; r++) {
            const uint8_t *p = data + lines[(size_t)r].p;
            uint32_t s0, s1, e;
            sam_field10(p, lines[(size_t)r].len, s0, s1, e);
            seq[(size_t)r] = Seq{p + s0, s1 - s0};
            hv[(size_t)r] = hash_bytes(p + s0, s1 - s0);
        }
    });
    for (int64_t b : bad) if (b >= 0) return c2b_sam_line_error(b >> 1, (int)(b & 1));
    std::unique_ptr<c2b_fastq> F(new c2b_fastq());
    F->n_reads = n_rec;
    dedup_records(seq, hv, n_rec, T, F.get(), [](const char *) {});
    *out = F.release();
    return C2B_OK;
}

// pass 2: every line of `text` whose field 10 is a unique read of the handle, as rstrip(line) + "\t" + annotation + "\n", in input
// order, appended to sam_path (the caller wrote the header); lines whose read is in no table are dropped
extern "C" int c2b_annotate_write_sam_passthrough(const c2b_annotation *a, const uint8_t *seqs, const int64_t *offsets, int64_t n_unique,
                                                  const uint8_t *text, size_t n_bytes, const char *sam_path, int32_t n_threads)
{
    if (!a || !sam_path || n_unique != a->n || (n_unique && !offsets) || (n_bytes && !text)) {
        g_fastq_err = "c2b_annotate_write_sam_passthrough: bad argument";
        return C2B_E_ARG;
    }
    std::vector<TLine> lines;
    split_text_lines(text, n_bytes, lines);
    const UniqueIndex idx(seqs, offsets, n_unique);
    const int64_t n_lines = (int64_t)lines.size();
    const int T = sam_threads(n_bytes, n_threads);
    std::vector<std::string> outs((size_t)T);
    std::vector<int64_t> bad((size_t)T, -1);
    run_threads(T, [&](int t) {
        const int64_t lo = n_lines * t / T, hi = n_lines * (t + 1) / T;
        bad[(size_t)t] = sam_first_bad(text, lines, (size_t)lo, (size_t)hi);
        if (bad[(size_t)t] >= 0) return;
        std::string &o = outs[(size_t)t];
        for (int64_t k = lo; k < hi; k++) {
            const uint8_t *p = text + lines[(size_t)k].p;
            uint32_t s0, s1, e;
            sam_field10(p, lines[(size_t)k].len, s0, s1, e);
            const int64_t u = idx.find(p + s0, s1 - s0);
            if (u < 0) continue;
            o.append((const char *)p, e);
            o.push_back('\t');
            o.append((const char *)a->ann.data() + a->ann_off[(size_t)u], (size_t)(a->ann_off[(size_t)u + 1] - a->ann_off[(size_t)u]));
            o.push_back('\n');
        }
    });
    for (int64_t b : bad) if (b >= 0) return c2b_sam_line_error(b >> 1, (int)(b & 1));
    if (!write_parts(sam_path, outs, std::string(), true)) {
        g_fastq_err = std::string("c2b_annotate_write_sam_passthrough: cannot write ") + sam_path;
        return C2B_E_STATE;
    }
    return C2B_OK;
}
