// c2b_fastq_gpu.cu -- FASTQ parse + exact de-duplication ON the GPU: the file's bytes cross PCIe once, the unique reads come
// back packed in first-seen order with their multiplicities (the same c2b_fastq object as the host front end, c2b_fastq.cpp).
//
// Also the pass-1 loop of process_bam (c2b_sam_dedup_gpu_buffer): the same passes over SAM text with one record per line and
// k_sam_records in place of k_records.
//
// Replaces: the FASTQ loop of process_fastq (reference: CRISPResso2/CRISPRessoCORE.py:1820-1849), same semantics as
// c2b_fastq_dedup -- text-mode universal newlines ("\n", "\r\n", a lone "\r"), a record starts at every fourth line that exists
// and takes the next three lines present or not, the sequence is line 2 stripped of ASCII whitespace, unique sequences in
// first-seen order -- at a rate closer to the one the alignment kernels consume reads at than the host front end reaches.
//
// Passes (one stream; CUB for the scans, the select and the sort):
//   k_count_ends / k_write_ends   line terminators per 4 KiB tile -> exclusive scan -> position of every line end
//   k_records                     one thread per record: line 4r+1, stripped -> (start, length, 64-bit hash)
//   k_sam_records                 (SAM) one warp per line: field 10 of the right-stripped line -> (start, length, hash)
//   k_dedup                       open-addressing table of record indices (CAS insert, byte-exact compare on a hash match): every
//                                 record finds its group's representative; atomicMin / atomicAdd give the group's first record
//                                 and its multiplicity -- exact, no probabilistic step
//   select + radix sort           representatives, ordered by their group's first record = first-seen order
//   k_emit                        packed sequences, offsets, counts, first indices
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <cuda_runtime.h>

#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <chrono>
#include <climits>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "c2b200.h"
#include "c2b_fastq_int.h"

namespace {

constexpr int TILE_T = 256, TILE_B = 16, TILE = TILE_T * TILE_B;       // bytes per block of the line-end passes

__device__ __forceinline__ bool is_space_d(uint8_t c) { return c == ' ' || (c >= 9 && c <= 13) || (c >= 0x1c && c <= 0x1f); }   // str.strip()

// byte p ends a line: '\n', or a '\r' that is not followed by '\n'
__device__ __forceinline__ bool line_end_at(const uint8_t *t, int64_t n, int64_t p)
{
    const uint8_t c = t[p];
    return c == '\n' || (c == '\r' && !(p + 1 < n && t[p + 1] == '\n'));
}

// line ends among the 16 bytes at `base` (a multiple of 16; the text buffer is 256-byte aligned): one 16-byte load and the byte
// after it instead of 17 byte loads -- bit k set = byte base + k ends a line
__device__ __forceinline__ uint32_t ends16(const uint8_t *__restrict__ t, int64_t n, int64_t base)
{
    if (base >= n) return 0u;
    uint32_t m = 0;
    if (base + 16 <= n) {
        const uint4 v = __ldg(reinterpret_cast<const uint4 *>(t + base));
        const uint32_t nxt = (base + 16 < n) ? (uint32_t)t[base + 16] : 0u;        // past the last byte: a final '\r' ends its line
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const uint32_t c = (w[k >> 2] >> (8 * (k & 3))) & 0xffu;
            const uint32_t d = (k < 15) ? ((w[(k + 1) >> 2] >> (8 * ((k + 1) & 3))) & 0xffu) : nxt;
            if (c == '\n' || (c == '\r' && d != '\n')) m |= 1u << k;
        }
        return m;
    }
    for (int k = 0; k < 16; k++) { const int64_t p = base + k; if (p < n && line_end_at(t, n, p)) m |= 1u << k; }
    return m;
}

__global__ void __launch_bounds__(TILE_T) k_count_ends(const uint8_t *__restrict__ t, int64_t n, int32_t *__restrict__ tile_count)
{
    static_assert(TILE_B == 16, "ends16 handles 16 bytes per thread");
    const int64_t base = (int64_t)blockIdx.x * TILE + (int64_t)threadIdx.x * TILE_B;
    const int c = __popc(ends16(t, n, base));
    typedef cub::BlockReduce<int, TILE_T> BR;
    __shared__ typename BR::TempStorage tmp;
    const int tot = BR(tmp).Sum(c);
    if (threadIdx.x == 0) tile_count[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(TILE_T) k_write_ends(const uint8_t *__restrict__ t, int64_t n, const int64_t *__restrict__ tile_off,
                                                      int64_t *__restrict__ ends)
{
    const int64_t base = (int64_t)blockIdx.x * TILE + (int64_t)threadIdx.x * TILE_B;
    uint32_t m = ends16(t, n, base);
    typedef cub::BlockScan<int, TILE_T> BS;
    __shared__ typename BS::TempStorage tmp;
    int pre;
    BS(tmp).ExclusiveSum(__popc(m), pre);
    int64_t o = tile_off[blockIdx.x] + pre;
    while (m) { ends[o++] = base + (__ffs(m) - 1); m &= m - 1; }              // ascending positions
}

// record r = lines 4r .. 4r+3; its sequence is line 4r+1 (absent: empty), stripped
__global__ void k_records(const uint8_t *__restrict__ t, int64_t n, const int64_t *__restrict__ ends, int64_t n_ends, int64_t n_lines,
                          int64_t n_rec, int64_t *__restrict__ rptr, int32_t *__restrict__ rlen, uint64_t *__restrict__ rhash)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rec) return;
    const int64_t L = 4 * r + 1;
    int64_t a = 0, b = 0;
    if (L < n_lines) {
        a = ends[L - 1] + 1;                                  // line L starts after the terminator of line L-1
        if (L < n_ends) { b = ends[L]; if (t[b] == '\n' && b > a && t[b - 1] == '\r') b--; }     // "\r\n": the '\r' belongs to the terminator
        else b = n;                                           // last line without a terminator
        while (a < b && is_space_d(t[a])) a++;
        while (b > a && is_space_d(t[b - 1])) b--;
    }
    uint64_t h = 0x9E3779B97F4A7C15ull ^ ((uint64_t)(b - a) * 0xff51afd7ed558ccdull);
    for (int64_t p = a; p < b; p++) { h = (h ^ t[p]) * 0x100000001b3ull; }
    h ^= h >> 29; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 32;
    rptr[r] = a; rlen[r] = (int32_t)(b - a); rhash[r] = h;
}

// SAM text (the pass-1 loop of process_bam, CRISPRessoCORE.py:2047-2057): record r = line r, its sequence is
// line.rstrip().split("\t")[9].  One warp per line, 32-byte windows: ballots of the tabs, of the non-space bytes (the rstrip end
// is one past the last of them) and of the non-ASCII bytes.  Field 10 starts after the 9th tab and ends at the 10th tab or at
// the rstrip end, whichever comes first; a 9th tab at or past the rstrip end means fewer than 10 fields (IndexError there).
// err: atomicMin of (line << 1) | kind over the bad lines, kind 0 = a non-ASCII byte, 1 = fewer than 10 fields.
// The hash is a sum of per-position terms (any function of the bytes serves: k_dedup decides equality by comparing bytes).
__global__ void __launch_bounds__(256) k_sam_records(const uint8_t *__restrict__ t, int64_t n, const int64_t *__restrict__ ends,
                                                     int64_t n_ends, int64_t n_rec, int64_t *__restrict__ rptr,
                                                     int32_t *__restrict__ rlen, uint64_t *__restrict__ rhash,
                                                     unsigned long long *__restrict__ err)
{
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= n_rec) return;
    const int64_t a = r ? ends[r - 1] + 1 : 0;
    int64_t b = n;
    if (r < n_ends) { b = ends[r]; if (t[b] == '\n' && b > a && t[b - 1] == '\r') b--; }
    int tabs = 0;
    int64_t p9 = -1, p10 = -1, last = a - 1;
    bool wide = false;
    for (int64_t w = a; w < b; w += 32) {
        const int64_t p = w + lane;
        const uint8_t c = p < b ? __ldg(t + p) : (uint8_t)' ';
        const uint32_t tb = __ballot_sync(0xffffffffu, c == '\t');
        const uint32_t ns = __ballot_sync(0xffffffffu, !is_space_d(c));
        wide |= __ballot_sync(0xffffffffu, c >= 0x80) != 0;
        if (ns) last = w + 31 - __clz(ns);
        const int pc = __popc(tb);
        if (p10 < 0 && tabs + pc >= 9) {                       // the 9th and / or 10th tab fall in this window
            uint32_t m = tb;
            for (int k = tabs; k < tabs + pc && k < 10; k++) {
                const int64_t q = w + __ffs(m) - 1;
                m &= m - 1;
                if (k == 8) p9 = q; else if (k == 9) p10 = q;
            }
        }
        tabs += pc;
    }
    const int64_t e = last + 1;                                 // rstrip end
    uint64_t h = 0;
    int64_t s0 = 0, s1 = 0;
    const bool shortl = p9 < 0 || p9 >= e;
    if (!wide && !shortl) {
        s0 = p9 + 1;
        s1 = (p10 >= 0 && p10 < e) ? p10 : e;
        for (int64_t p = s0 + lane; p < s1; p += 32) {
            uint64_t x = ((uint64_t)__ldg(t + p) << 40) ^ (uint64_t)(p - s0);
            x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 29;
            h += x;
        }
        for (int d = 16; d; d >>= 1) h += __shfl_xor_sync(0xffffffffu, h, d);
        h ^= (uint64_t)(s1 - s0) * 0x9E3779B97F4A7C15ull;
        h ^= h >> 31; h *= 0xff51afd7ed558ccdull; h ^= h >> 32;
    }
    if (lane == 0) {
        if (wide || shortl) atomicMin(err, ((unsigned long long)r << 1) | (wide ? 0ull : 1ull));
        rptr[r] = s0; rlen[r] = (int32_t)(s1 - s0); rhash[r] = h;
    }
}

__global__ void k_dedup(const uint8_t *__restrict__ t, const int64_t *__restrict__ rptr, const int32_t *__restrict__ rlen,
                        const uint64_t *__restrict__ rhash, int64_t n_rec, int32_t *__restrict__ table, uint32_t mask,
                        int32_t *__restrict__ first, int32_t *__restrict__ count, uint8_t *__restrict__ is_rep)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rec) return;
    const uint64_t h = rhash[r];
    const int32_t len = rlen[r];
    const uint8_t *me = t + rptr[r];
    uint32_t slot = (uint32_t)(h >> 17) & mask;
    int32_t rep = -1;
    bool mine = false;
    for (;;) {
        int32_t cur = table[slot];
        if (cur < 0) {
            const int32_t old = atomicCAS(&table[slot], -1, (int32_t)r);
            if (old < 0) { rep = (int32_t)r; mine = true; break; }
            cur = old;
        }
        if (rhash[cur] == h && rlen[cur] == len) {            // byte-exact compare: equality is never decided by the hash
            const uint8_t *o = t + rptr[cur];
            bool same = true;
            for (int32_t k = 0; k < len; k++) if (o[k] != me[k]) { same = false; break; }
            if (same) { rep = cur; break; }
        }
        slot = (slot + 1) & mask;
    }
    is_rep[r] = mine ? 1 : 0;
    atomicMin(&first[rep], (int32_t)r);
    atomicAdd(&count[rep], 1);
}

__global__ void k_gather_first(const int32_t *__restrict__ reps, const int32_t *__restrict__ first, int64_t nu, int32_t *__restrict__ keys)
{
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u < nu) keys[u] = first[reps[u]];
}

__global__ void k_lens(const int32_t *__restrict__ reps_sorted, const int32_t *__restrict__ rlen, int64_t nu, int64_t *__restrict__ lens)
{
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u < nu) lens[u] = rlen[reps_sorted[u]];
}

// one warp per unique read
__global__ void k_emit(const uint8_t *__restrict__ t, const int32_t *__restrict__ reps_sorted, const int64_t *__restrict__ rptr,
                       const int32_t *__restrict__ rlen, const int32_t *__restrict__ first, const int32_t *__restrict__ count,
                       const int64_t *__restrict__ offs, int64_t nu, uint8_t *__restrict__ seqs, int32_t *__restrict__ o_count,
                       int64_t *__restrict__ o_first)
{
    const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (u >= nu) return;
    const int32_t rep = reps_sorted[u];
    const uint8_t *src = t + rptr[rep];
    uint8_t *dst = seqs + offs[u];
    const int32_t len = rlen[rep];
    for (int32_t k = lane; k < len; k += 32) dst[k] = src[k];
    if (lane == 0) { o_count[u] = count[rep]; o_first[u] = first[rep]; }
}

// stream-ordered allocations from the device's default pool: blocks released by one call are re-used by the next without a
// trip to the driver (the pool keeps up to POOL_KEEP bytes between calls)
constexpr uint64_t POOL_KEEP = 4ull << 30;
thread_local cudaStream_t g_alloc_stream = nullptr;
struct DBuf {
    void *p = nullptr;
    cudaStream_t s = nullptr;
    ~DBuf() { if (p) cudaFreeAsync(p, s); }
    cudaError_t get(size_t n) { s = g_alloc_stream; return cudaMallocAsync(&p, n ? n : 16, s); }
    void drop() { if (p) { cudaFreeAsync(p, s); p = nullptr; } }
    template <class T> T *as() { return (T *)p; }
};

#define GCHK(call) do { cudaError_t _r = (call); if (_r != cudaSuccess) { c2b_fastq_set_error(std::string("c2b_fastq_dedup_gpu: " #call ": ") + cudaGetErrorString(_r)); return C2B_E_CUDA; } } while (0)

// Pinned ring for the host <-> device byte streams.  Worker threads move slices of each block between the caller's memory
// (page-cache pages of the file / the result arrays) and the ring while the copy engine moves the neighbouring block, so the
// slower of the two sets the pace; the workers live for one transfer (no thread start per block).
struct Ring {
    static constexpr int NB = 3;
    static constexpr size_t CH = 32u << 20;
    uint8_t *p[NB] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev[NB] = {nullptr, nullptr, nullptr};
    std::mutex mu;                                            // one transfer at a time through the ring
    ~Ring() { for (int k = 0; k < NB; k++) { if (p[k]) cudaFreeHost(p[k]); if (ev[k]) cudaEventDestroy(ev[k]); } }
    cudaError_t ensure()
    {
        for (int k = 0; k < NB; k++) {
            if (!p[k]) { cudaError_t r = cudaHostAlloc((void **)&p[k], CH, cudaHostAllocDefault); if (r != cudaSuccess) { p[k] = nullptr; return r; } }
            if (!ev[k]) { cudaError_t r = cudaEventCreateWithFlags(&ev[k], cudaEventDisableTiming); if (r != cudaSuccess) { ev[k] = nullptr; return r; } }
        }
        return cudaSuccess;
    }
};
Ring g_ring;

int ring_threads(size_t n)
{
    if (n < (8u << 20)) return 1;
    unsigned hc = std::thread::hardware_concurrency();
    return (int)std::max(2u, std::min(16u, hc ? hc / 2 : 8u));
}

// host -> device: fill(dst, offset, len) writes bytes [offset, offset + len) of the source into dst
template <class Fill> int ring_h2d(uint8_t *d_dst, size_t n, cudaStream_t s, Fill fill)
{
    std::lock_guard<std::mutex> lk(g_ring.mu);
    GCHK(g_ring.ensure());
    const size_t CH = Ring::CH;
    const int NB = Ring::NB;
    const int64_t nch = (int64_t)((n + CH - 1) / CH);
    const int T = ring_threads(n);
    std::vector<std::atomic<int>> filled((size_t)nch);
    for (auto &f : filled) f.store(0);
    std::atomic<int64_t> avail(NB);                           // blocks [0, avail) may be filled
    std::atomic<bool> stop(false);
    auto worker = [&](int t) {
        for (int64_t c = 0; c < nch && !stop.load(std::memory_order_relaxed); c++) {
            while (avail.load(std::memory_order_acquire) <= c) { if (stop.load(std::memory_order_relaxed)) return; std::this_thread::yield(); }
            const size_t o = (size_t)c * CH, m = std::min(CH, n - o);
            const size_t a = m * (size_t)t / T, b = m * (size_t)(t + 1) / T;
            if (b > a) fill(g_ring.p[c % NB] + a, o + a, b - a);
            filled[(size_t)c].fetch_add(1, std::memory_order_release);
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(worker, t);
    cudaError_t err = cudaSuccess;
    if (T == 1) {
        for (int64_t c = 0; c < nch && err == cudaSuccess; c++) {
            const size_t o = (size_t)c * CH, m = std::min(CH, n - o);
            if (c >= NB) err = cudaEventSynchronize(g_ring.ev[c % NB]);
            if (err != cudaSuccess) break;
            fill(g_ring.p[c % NB], o, m);
            err = cudaMemcpyAsync(d_dst + o, g_ring.p[c % NB], m, cudaMemcpyHostToDevice, s);
            if (err == cudaSuccess) err = cudaEventRecord(g_ring.ev[c % NB], s);
        }
    } else {
        // this thread drives the copy engine; slice 0 is filled by a helper so that the driver never waits behind a memcpy
        th.emplace_back(worker, 0);
        for (int64_t c = 0; c < nch; c++) {
            while (filled[(size_t)c].load(std::memory_order_acquire) < T) std::this_thread::yield();
            const size_t o = (size_t)c * CH, m = std::min(CH, n - o);
            err = cudaMemcpyAsync(d_dst + o, g_ring.p[c % NB], m, cudaMemcpyHostToDevice, s);
            if (err == cudaSuccess) err = cudaEventRecord(g_ring.ev[c % NB], s);
            if (err == cudaSuccess) err = cudaEventSynchronize(g_ring.ev[c % NB]);      // helpers are already filling the next blocks
            if (err != cudaSuccess) break;
            avail.store(c + NB + 1, std::memory_order_release);
        }
    }
    stop.store(err != cudaSuccess);
    for (auto &x : th) x.join();
    GCHK(err);
    return C2B_OK;
}

// device -> host: the copy engine fills ring blocks, the helpers scatter them into dst (first touch of dst's pages in parallel)
int ring_d2h(uint8_t *dst, const uint8_t *d_src, size_t n, cudaStream_t s)
{
    if (n == 0) return C2B_OK;
    std::lock_guard<std::mutex> lk(g_ring.mu);
    GCHK(g_ring.ensure());
    const size_t CH = Ring::CH;
    const int NB = Ring::NB;
    const int64_t nch = (int64_t)((n + CH - 1) / CH);
    const int T = ring_threads(n);
    if (T == 1) {
        for (int64_t c = 0; c < nch; c++) {
            const size_t o = (size_t)c * CH, m = std::min(CH, n - o);
            GCHK(cudaMemcpyAsync(g_ring.p[0], d_src + o, m, cudaMemcpyDeviceToHost, s));
            GCHK(cudaStreamSynchronize(s));
            memcpy(dst + o, g_ring.p[0], m);
        }
        return C2B_OK;
    }
    std::vector<std::atomic<int>> drained((size_t)nch);
    for (auto &f : drained) f.store(0);
    std::atomic<int64_t> ready(0);                            // blocks [0, ready) sit in the ring
    std::atomic<bool> stop(false);
    auto worker = [&](int t) {
        for (int64_t c = 0; c < nch; c++) {
            while (ready.load(std::memory_order_acquire) <= c) { if (stop.load(std::memory_order_relaxed)) return; std::this_thread::yield(); }
            const size_t o = (size_t)c * CH, m = std::min(CH, n - o);
            const size_t a = m * (size_t)t / T, b = m * (size_t)(t + 1) / T;
            if (b > a) memcpy(dst + o + a, g_ring.p[c % NB] + a, b - a);
            drained[(size_t)c].fetch_add(1, std::memory_order_release);
        }
    };
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++) th.emplace_back(worker, t);
    cudaError_t err = cudaSuccess;
    for (int64_t c = 0; c < nch; c++) {
        if (c >= NB) while (drained[(size_t)(c - NB)].load(std::memory_order_acquire) < T) std::this_thread::yield();
        const size_t o = (size_t)c * CH, m = std::min(CH, n - o);
        err = cudaMemcpyAsync(g_ring.p[c % NB], d_src + o, m, cudaMemcpyDeviceToHost, s);
        if (err == cudaSuccess) err = cudaStreamSynchronize(s);
        if (err != cudaSuccess) break;
        ready.store(c + 1, std::memory_order_release);
    }
    if (err != cudaSuccess) stop.store(true);
    for (auto &x : th) x.join();
    GCHK(err);
    return C2B_OK;
}

// where the FASTQ text comes from: memory (buffer entry, inflated gzip) or a file descriptor read with pread (no page faults
// of a mapping on the way into the ring)
struct Source {
    const uint8_t *mem = nullptr;
    int fd = -1;
    bool read(uint8_t *dst, size_t off, size_t len) const
    {
        if (mem) { memcpy(dst, mem + off, len); return true; }
        while (len) {
            const ssize_t r = pread(fd, dst, len, (off_t)off);
            if (r <= 0) return false;
            dst += r; off += (size_t)r; len -= (size_t)r;
        }
        return true;
    }
};

// sam = false: FASTQ records (k_records); true: one SAM line per record (k_sam_records)
int dedup_device(const Source &src, size_t n, int device, c2b_fastq **out, bool sam = false)
{
    const bool verbose = getenv("C2B_FASTQ_VERBOSE") != nullptr;
    auto t_last = std::chrono::steady_clock::now();
    auto lap = [&](const char *what) {
        if (!verbose) return;
        cudaDeviceSynchronize();
        auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[c2b_fastq_gpu] %-10s %.4f s\n", what, std::chrono::duration<double>(now - t_last).count());
        t_last = now;
    };
    GCHK(cudaSetDevice(device));
    c2b_fastq *F = new c2b_fastq();
    std::unique_ptr<c2b_fastq> guard(F);
    if (n == 0) { F->offsets.assign(1, 0); F->seqs.reset(new uint8_t[16]); *out = guard.release(); return C2B_OK; }
    if (n >= ((size_t)1 << 40)) { c2b_fastq_set_error("c2b_fastq_dedup_gpu: file too large"); return C2B_E_LIMIT; }
    cudaStream_t s;
    GCHK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    struct SG { cudaStream_t s; ~SG() { cudaStreamSynchronize(s); cudaStreamDestroy(s); } } sg{s};
    g_alloc_stream = s;
    {
        cudaMemPool_t pool;
        uint64_t keep = POOL_KEEP;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    DBuf d_text, d_tc, d_to, d_ends, d_tmp;
    GCHK(d_text.get(n + 16));
    lap("alloc");
    std::atomic<bool> short_read(false);
    int rc = ring_h2d(d_text.as<uint8_t>(), n, s, [&](uint8_t *dst, size_t off, size_t len) { if (!src.read(dst, off, len)) short_read.store(true); });
    if (rc) return rc;
    if (short_read.load()) { c2b_fastq_set_error("c2b_fastq_dedup_gpu: short read from the file"); return C2B_E_ARG; }
    lap("upload");
    const int64_t ntiles = (int64_t)((n + TILE - 1) / TILE);
    GCHK(d_tc.get((size_t)ntiles * 4));
    GCHK(d_to.get((size_t)(ntiles + 1) * 8));
    k_count_ends<<<(unsigned)ntiles, TILE_T, 0, s>>>(d_text.as<uint8_t>(), (int64_t)n, d_tc.as<int32_t>());
    size_t tb = 0;
    GCHK(cub::DeviceScan::ExclusiveSum(nullptr, tb, d_tc.as<int32_t>(), d_to.as<int64_t>(), (int)ntiles, s));
    size_t tmp_cap = tb + 256;
    GCHK(d_tmp.get(tmp_cap));
    GCHK(cub::DeviceScan::ExclusiveSum(d_tmp.p, tb, d_tc.as<int32_t>(), d_to.as<int64_t>(), (int)ntiles, s));
    int64_t last_off = 0; int32_t last_cnt = 0; uint8_t last_byte = 0;
    GCHK(cudaMemcpyAsync(&last_off, d_to.as<int64_t>() + (ntiles - 1), 8, cudaMemcpyDeviceToHost, s));
    GCHK(cudaMemcpyAsync(&last_cnt, d_tc.as<int32_t>() + (ntiles - 1), 4, cudaMemcpyDeviceToHost, s));
    GCHK(cudaStreamSynchronize(s));
    if (!src.read(&last_byte, n - 1, 1)) { c2b_fastq_set_error("c2b_fastq_dedup_gpu: short read from the file"); return C2B_E_ARG; }
    const int64_t n_ends = last_off + last_cnt;
    const bool open_tail = !(last_byte == '\n' || last_byte == '\r');             // the last line has no terminator
    const int64_t n_lines = n_ends + (open_tail ? 1 : 0);
    const int64_t n_rec = sam ? n_lines : (n_lines + 3) / 4;
    if (n_rec >= (int64_t)INT_MAX / 2) { c2b_fastq_set_error("c2b_fastq_dedup_gpu: more than 2^30 records"); return C2B_E_LIMIT; }
    GCHK(d_ends.get((size_t)(n_ends + 1) * 8));
    k_write_ends<<<(unsigned)ntiles, TILE_T, 0, s>>>(d_text.as<uint8_t>(), (int64_t)n, d_to.as<int64_t>(), d_ends.as<int64_t>());
    lap("lines");
    F->n_reads = n_rec;
    if (n_rec == 0) { F->offsets.assign(1, 0); F->seqs.reset(new uint8_t[16]); *out = guard.release(); return C2B_OK; }
    DBuf d_ptr, d_len, d_hash, d_table, d_first, d_count, d_isrep, d_reps, d_nsel, d_keys, d_keys2, d_reps2, d_lens, d_offs;
    GCHK(d_ptr.get((size_t)n_rec * 8)); GCHK(d_len.get((size_t)n_rec * 4)); GCHK(d_hash.get((size_t)n_rec * 8));
    const unsigned TB = 256, GB = (unsigned)((n_rec + TB - 1) / TB);
    if (!sam) {
        // line L - 1 of record 0 is line 0: ends[L - 1] is read for L >= 1 only, which k_records guarantees (L = 4r + 1 >= 1)
        k_records<<<GB, TB, 0, s>>>(d_text.as<uint8_t>(), (int64_t)n, d_ends.as<int64_t>(), n_ends, n_lines, n_rec, d_ptr.as<int64_t>(),
                                    d_len.as<int32_t>(), d_hash.as<uint64_t>());
    } else {
        DBuf d_err;
        GCHK(d_err.get(8));
        GCHK(cudaMemsetAsync(d_err.p, 0xff, 8, s));
        k_sam_records<<<(unsigned)((n_rec * 32 + TB - 1) / TB), TB, 0, s>>>(d_text.as<uint8_t>(), (int64_t)n, d_ends.as<int64_t>(), n_ends,
                                                                            n_rec, d_ptr.as<int64_t>(), d_len.as<int32_t>(),
                                                                            d_hash.as<uint64_t>(), d_err.as<unsigned long long>());
        unsigned long long bad = ~0ull;
        GCHK(cudaMemcpyAsync(&bad, d_err.p, 8, cudaMemcpyDeviceToHost, s));
        GCHK(cudaStreamSynchronize(s));
        if (bad != ~0ull) return c2b_sam_line_error((int64_t)(bad >> 1), (int)(bad & 1));
    }
    uint32_t cap = 64;
    while ((int64_t)cap < 2 * n_rec + 8) cap <<= 1;
    GCHK(d_table.get((size_t)cap * 4)); GCHK(d_first.get((size_t)n_rec * 4)); GCHK(d_count.get((size_t)n_rec * 4)); GCHK(d_isrep.get((size_t)n_rec));
    GCHK(cudaMemsetAsync(d_table.p, 0xff, (size_t)cap * 4, s));
    GCHK(cudaMemsetAsync(d_first.p, 0x7f, (size_t)n_rec * 4, s));              // 0x7f7f7f7f: above every record index
    GCHK(cudaMemsetAsync(d_count.p, 0, (size_t)n_rec * 4, s));
    k_dedup<<<GB, TB, 0, s>>>(d_text.as<uint8_t>(), d_ptr.as<int64_t>(), d_len.as<int32_t>(), d_hash.as<uint64_t>(), n_rec, d_table.as<int32_t>(),
                              cap - 1, d_first.as<int32_t>(), d_count.as<int32_t>(), d_isrep.as<uint8_t>());
    lap("dedup");
    // representatives, then their order by first record
    GCHK(d_reps.get((size_t)n_rec * 4)); GCHK(d_nsel.get(8));
    thrust::counting_iterator<int32_t> iota(0);
    size_t b1 = 0, b2 = 0;
    GCHK(cub::DeviceSelect::Flagged(nullptr, b1, iota, d_isrep.as<uint8_t>(), d_reps.as<int32_t>(), d_nsel.as<int32_t>(), (int)n_rec, s));
    if (b1 + 256 > tmp_cap) { d_tmp.drop(); tmp_cap = b1 + 256; GCHK(d_tmp.get(tmp_cap)); }
    GCHK(cub::DeviceSelect::Flagged(d_tmp.p, b1, iota, d_isrep.as<uint8_t>(), d_reps.as<int32_t>(), d_nsel.as<int32_t>(), (int)n_rec, s));
    int32_t nu32 = 0;
    GCHK(cudaMemcpyAsync(&nu32, d_nsel.p, 4, cudaMemcpyDeviceToHost, s));
    GCHK(cudaStreamSynchronize(s));
    const int64_t nu = nu32;
    GCHK(d_keys.get((size_t)nu * 4)); GCHK(d_keys2.get((size_t)nu * 4)); GCHK(d_reps2.get((size_t)nu * 4));
    const unsigned GU = (unsigned)((nu + TB - 1) / TB);
    k_gather_first<<<GU, TB, 0, s>>>(d_reps.as<int32_t>(), d_first.as<int32_t>(), nu, d_keys.as<int32_t>());
    GCHK(cub::DeviceRadixSort::SortPairs(nullptr, b2, d_keys.as<int32_t>(), d_keys2.as<int32_t>(), d_reps.as<int32_t>(), d_reps2.as<int32_t>(), (int)nu, 0, 32, s));
    if (b2 + 256 > tmp_cap) { d_tmp.drop(); tmp_cap = b2 + 256; GCHK(d_tmp.get(tmp_cap)); }
    GCHK(cub::DeviceRadixSort::SortPairs(d_tmp.p, b2, d_keys.as<int32_t>(), d_keys2.as<int32_t>(), d_reps.as<int32_t>(), d_reps2.as<int32_t>(), (int)nu, 0, 32, s));
    GCHK(d_lens.get((size_t)(nu + 1) * 8)); GCHK(d_offs.get((size_t)(nu + 1) * 8));
    GCHK(cudaMemsetAsync(d_lens.p, 0, (size_t)(nu + 1) * 8, s));
    k_lens<<<GU, TB, 0, s>>>(d_reps2.as<int32_t>(), d_len.as<int32_t>(), nu, d_lens.as<int64_t>());
    size_t b3 = 0;
    GCHK(cub::DeviceScan::ExclusiveSum(nullptr, b3, d_lens.as<int64_t>(), d_offs.as<int64_t>(), (int)(nu + 1), s));
    if (b3 + 256 > tmp_cap) { d_tmp.drop(); tmp_cap = b3 + 256; GCHK(d_tmp.get(tmp_cap)); }
    GCHK(cub::DeviceScan::ExclusiveSum(d_tmp.p, b3, d_lens.as<int64_t>(), d_offs.as<int64_t>(), (int)(nu + 1), s));
    int64_t tot = 0;
    GCHK(cudaMemcpyAsync(&tot, d_offs.as<int64_t>() + nu, 8, cudaMemcpyDeviceToHost, s));
    GCHK(cudaStreamSynchronize(s));
    DBuf d_seqs, d_ocount, d_ofirst;
    GCHK(d_seqs.get((size_t)tot + 16)); GCHK(d_ocount.get((size_t)nu * 4)); GCHK(d_ofirst.get((size_t)nu * 8));
    k_emit<<<(unsigned)((nu * 32 + TB - 1) / TB), TB, 0, s>>>(d_text.as<uint8_t>(), d_reps2.as<int32_t>(), d_ptr.as<int64_t>(), d_len.as<int32_t>(),
                                                             d_first.as<int32_t>(), d_count.as<int32_t>(), d_offs.as<int64_t>(), nu, d_seqs.as<uint8_t>(),
                                                             d_ocount.as<int32_t>(), d_ofirst.as<int64_t>());
    lap("emit");
    F->offsets.resize((size_t)nu + 1); F->counts.resize((size_t)nu); F->first_index.resize((size_t)nu);
    F->seqs.reset(new uint8_t[(size_t)tot + 16]);
    GCHK(cudaStreamSynchronize(s));
    GCHK(cudaGetLastError());
    if ((rc = ring_d2h((uint8_t *)F->offsets.data(), d_offs.as<uint8_t>(), (size_t)(nu + 1) * 8, s))) return rc;
    if ((rc = ring_d2h((uint8_t *)F->counts.data(), d_ocount.as<uint8_t>(), (size_t)nu * 4, s))) return rc;
    if ((rc = ring_d2h((uint8_t *)F->first_index.data(), d_ofirst.as<uint8_t>(), (size_t)nu * 8, s))) return rc;
    if ((rc = ring_d2h(F->seqs.get(), d_seqs.as<uint8_t>(), (size_t)tot, s))) return rc;
    int32_t mx = 0;
    for (int64_t u = 0; u < nu; u++) mx = std::max<int32_t>(mx, (int32_t)(F->offsets[(size_t)u + 1] - F->offsets[(size_t)u]));
    F->max_len = mx;
    lap("download");
    *out = guard.release();
    return C2B_OK;
}

}  // namespace

extern "C" int c2b_fastq_gpu_available(void) { return 1; }

extern "C" int c2b_fastq_dedup_gpu_buffer(const uint8_t *data, size_t n, int32_t device, c2b_fastq **out)
{
    if (!out || (n && !data)) return C2B_E_ARG;
    *out = nullptr;
    Source src;
    src.mem = data;
    return dedup_device(src, n, device, out);
}

extern "C" int c2b_sam_dedup_gpu_buffer(const uint8_t *data, size_t n, int32_t device, c2b_fastq **out)
{
    if (!out || (n && !data)) return C2B_E_ARG;
    *out = nullptr;
    Source src;
    src.mem = data;
    return dedup_device(src, n, device, out, true);
}

extern "C" int c2b_fastq_dedup_gpu(const char *path, int32_t device, c2b_fastq **out)
{
    if (!path || !out) return C2B_E_ARG;
    *out = nullptr;
    const size_t L = strlen(path);
    if (L > 3 && strcmp(path + L - 3, ".gz") == 0) {          // gzip: one inflate stream on the host, then the same device passes
        c2b_bytes buf;
        std::string err;
        if (!c2b_fastq_read_gz(path, buf, err)) { c2b_fastq_set_error("c2b_fastq_dedup_gpu: " + err); return C2B_E_ARG; }
        Source src;
        src.mem = buf.data();
        return dedup_device(src, buf.size(), device, out);
    }
    int fd = open(path, O_RDONLY);
    if (fd < 0) { c2b_fastq_set_error(std::string("c2b_fastq_dedup_gpu: cannot open ") + path); return C2B_E_ARG; }
    struct stat st;
    if (fstat(fd, &st) != 0) { close(fd); c2b_fastq_set_error("c2b_fastq_dedup_gpu: cannot stat file"); return C2B_E_ARG; }
    Source src;
    src.fd = fd;
    posix_fadvise(fd, 0, 0, POSIX_FADV_SEQUENTIAL);
    const int rc = dedup_device(src, (size_t)st.st_size, device, out);
    close(fd);
    return rc;
}
