// c2b_alleles.cpp -- native allele-level consumers of the engine's unique-read table (host code, no CUDA).
//
// Replaces, for one run's alignments held in the engine's compact form (op streams + meta words + packed reads):
//   * the allele table of CRISPRessoCORE.py:3909-3959 (get_allele_row per variant), :4298-4303 (DataFrame, %Reads, sort by
//     #Reads desc, Aligned_Sequence, Reference_Sequence) and the text of Alleles_frequency_table.txt (:4498-4535,
//     DataFrame.to_csv(sep='\t', index=None) of the nine crispresso2Cols columns);
//   * CRISPRessoShared.get_dataframe_around_cut_asymmetrical / get_dataframe_around_cut (CRISPRessoShared.py:1513-1531):
//     per allele the window [cut_idx - left + 1, cut_idx + right + 1) of both aligned strings (cut_idx = the column that holds
//     reference position cut_point, i.e. row['ref_positions'].index(cut_point)), pandas groupby(...).sum() over the six key
//     columns and the final sort -- the grouping, with its Kahan sum and sort, shared with the --base_editor_output quilt table
//     (c2b_group_around_cut, called by c2b_be_quilt_table in c2b_engine.cu).
// Nothing here aligns or classifies: rows arrive with their alignment (ops) and their per-read numbers (n_deleted, ...,
// Read_Status) as the GPU produced them; this file spells strings, sorts, groups and formats -- the work pandas does row by
// row in the reference (10 % of a reference run's time, SURVEY.md section 8f rank 2).
//
// Float parity: %Reads of an around-cut group is the sum of its rows' %Reads in row order with pandas' Kahan-compensated
// group_sum (pandas/_libs/groupby.pyx), restated in group_add(); no multiplication is involved, so FP contraction cannot
// change it.  %Reads text in the frequency table is supplied by the caller (repr() of the few distinct values).
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "c2b200.h"
#include "c2b_fastq_int.h"

namespace {

constexpr int OP_M = 0, OP_J = 1, OP_I = 2, OP_NONE = 3;

}  // namespace

struct c2b_alleles {
    int64_t n = 0;
    std::vector<uint8_t> arena;            // row i: aligned read at arena[off[i]], aligned reference at arena[off[i] + len[i]]
    std::vector<int64_t> off;              // n + 1
    std::vector<int32_t> len;              // alignment columns of row i
    std::vector<int64_t> count;
    std::vector<int64_t> order;            // rows sorted by (#Reads desc, Aligned_Sequence, Reference_Sequence), stable
    // result of the last c2b_alleles_around_cut
    std::vector<c2b_cut_group> groups;       // window strings point into arena
    int32_t win_max = 0;
    std::string err;
};

static int nthreads(int32_t req, int64_t n, int64_t grain)
{
    int t = req > 0 ? req : (int)std::max(1u, std::thread::hardware_concurrency());
    t = (int)std::min<int64_t>(t, std::max<int64_t>(1, n / grain));
    return std::min(t, 64);
}

template <class F>
static void parallel_for(int T, F f)
{
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(f, t);
    f(0);
    for (auto &x : th) x.join();
}

static inline int cmp_rows(const c2b_alleles &A, int64_t a, int64_t b)
{
    if (A.count[a] != A.count[b]) return A.count[a] > A.count[b] ? -1 : 1;
    // Python str comparison of ASCII text = byte order, shorter prefix first; Aligned_Sequence, then Reference_Sequence
    for (int part = 0; part < 2; part++) {
        const uint8_t *pa = A.arena.data() + A.off[a] + (part ? A.len[a] : 0), *pb = A.arena.data() + A.off[b] + (part ? A.len[b] : 0);
        const int la = A.len[a], lb = A.len[b];
        const int c = memcmp(pa, pb, (size_t)std::min(la, lb));
        if (c) return c < 0 ? -1 : 1;
        if (la != lb) return la < lb ? -1 : 1;
    }
    return 0;
}

extern "C" {

int c2b_alleles_build(const uint8_t *reads, const int64_t *offsets, const uint64_t *ops, const uint32_t *meta, int32_t NW,
                      int64_t n_rows, const int64_t *row_read, const int64_t *row_slot, const int32_t *row_ref,
                      const int64_t *row_count, int32_t n_refs, const char *const *ref_seqs, const int32_t *ref_lens,
                      const uint8_t *comp256, int32_t n_threads, c2b_alleles **out)
{
    if (!out) return C2B_E_ARG;
    *out = nullptr;
    if (n_rows < 0 || (n_rows && (!reads || !offsets || !ops || !meta || !row_read || !row_slot || !row_ref || !row_count)) ||
        NW < 1 || n_refs < 1 || !ref_seqs || !ref_lens || !comp256) return C2B_E_ARG;
    c2b_alleles *A = new c2b_alleles();
    A->n = n_rows;
    A->off.assign((size_t)n_rows + 1, 0);
    A->len.assign((size_t)n_rows, 0);
    A->count.assign(row_count, row_count + n_rows);
    for (int64_t i = 0; i < n_rows; i++) {
        const uint32_t m = meta[row_slot[i]];
        const int n = (int)(m & 0xffffu);
        if (n < 1 || n > 32 * NW || row_ref[i] < 0 || row_ref[i] >= n_refs) { delete A; return C2B_E_ARG; }
        A->len[(size_t)i] = n;
        A->off[(size_t)i + 1] = A->off[(size_t)i] + 2 * (int64_t)n;
    }
    A->arena.resize((size_t)A->off[(size_t)n_rows] + 16);
    const int T = nthreads(n_threads, n_rows, 2048);
    std::vector<int> bad((size_t)T, 0);
    parallel_for(T, [&](int t) {                           // spell the two aligned strings of every row (Align.pyx:422-434)
        const int64_t lo = n_rows * t / T, hi = n_rows * (t + 1) / T;
        for (int64_t r = lo; r < hi; r++) {
            const uint32_t m = meta[row_slot[r]];
            const int n = (int)(m & 0xffffu), strand = (int)((m >> 16) & 1u);
            const uint64_t *o = ops + row_slot[r] * (int64_t)NW;
            const uint8_t *rd = reads + offsets[row_read[r]];
            const int J = (int)(offsets[row_read[r] + 1] - offsets[row_read[r]]);
            const char *rf = ref_seqs[row_ref[r]];
            int i = ref_lens[row_ref[r]], j = J;
            uint8_t *o_read = A->arena.data() + A->off[(size_t)r], *o_ref = o_read + n;
            bool ok = true;
            for (int q = 0; q < n; q++) {                  // column q from the right end
                const int op = (int)((o[q >> 5] >> (2 * (q & 31))) & 3ull);
                uint8_t a = '-', b = '-';
                if (op == OP_NONE) { ok = false; break; }
                if (op != OP_J) { if (j < 1) { ok = false; break; } j--; a = strand ? comp256[rd[J - 1 - j]] : rd[j]; }
                if (op != OP_I) { if (i < 1) { ok = false; break; } i--; b = (uint8_t)rf[i]; }
                o_read[n - 1 - q] = a; o_ref[n - 1 - q] = b;
            }
            if (!ok || i != 0 || j != 0) bad[(size_t)t]++;
        }
    });
    for (int b : bad) if (b) { delete A; return C2B_E_ARG; }
    // order: stable merge sort, chunks sorted on threads, then merged pairwise
    A->order.resize((size_t)n_rows);
    for (int64_t i = 0; i < n_rows; i++) A->order[(size_t)i] = i;
    auto less = [&](int64_t a, int64_t b) { return cmp_rows(*A, a, b) < 0; };
    int C = 1; while (C < T) C <<= 1;
    if (n_rows < 4096) C = 1;
    std::vector<int64_t> cut((size_t)C + 1);
    for (int c = 0; c <= C; c++) cut[(size_t)c] = n_rows * c / C;
    parallel_for(std::min(T, C), [&](int t) {
        for (int c = t; c < C; c += std::min(T, C)) std::stable_sort(A->order.begin() + cut[(size_t)c], A->order.begin() + cut[(size_t)c + 1], less);
    });
    std::vector<int64_t> tmp((size_t)n_rows);
    for (int w = 1; w < C; w <<= 1) {
        const int pairs = C / (2 * w);
        parallel_for(std::min(T, pairs), [&](int t) {
            for (int p = t; p < pairs; p += std::min(T, pairs)) {
                const int64_t a = cut[(size_t)(2 * w * p)], m = cut[(size_t)(2 * w * p + w)], b = cut[(size_t)(2 * w * p + 2 * w)];
                std::merge(A->order.begin() + a, A->order.begin() + m, A->order.begin() + m, A->order.begin() + b, tmp.begin() + a, less);   // stable: left run first on ties
                std::copy(tmp.begin() + a, tmp.begin() + b, A->order.begin() + a);
            }
        });
    }
    *out = A;
    return C2B_OK;
}

void c2b_alleles_free(c2b_alleles *A) { delete A; }
int64_t c2b_alleles_n(const c2b_alleles *A) { return A ? A->n : 0; }
const int64_t *c2b_alleles_order(const c2b_alleles *A) { return A ? A->order.data() : nullptr; }
const uint8_t *c2b_alleles_arena(const c2b_alleles *A) { return A ? A->arena.data() : nullptr; }
const int64_t *c2b_alleles_offsets(const c2b_alleles *A) { return A ? A->off.data() : nullptr; }
const int32_t *c2b_alleles_lengths(const c2b_alleles *A) { return A ? A->len.data() : nullptr; }

// Alleles_frequency_table.txt: header + one line per row of `rows` (normally the sorted order), tab-separated:
// Aligned_Sequence Reference_Sequence Reference_Name Read_Status n_deleted n_inserted n_mutated #Reads %Reads
// name_id / status_id / pct_id index the caller's string tables (a handful of distinct values each).
int c2b_alleles_write_tsv(const c2b_alleles *A, const char *path, int64_t n_sel, const int64_t *rows,
                          const int32_t *name_id, const char *const *names, const int32_t *status_id, const char *const *statuses,
                          const int32_t *n_deleted, const int32_t *n_inserted, const int32_t *n_mutated,
                          const int32_t *pct_id, const char *const *pcts, int32_t n_threads)
{
    if (!A || !path || n_sel < 0 || (n_sel && (!rows || !name_id || !names || !status_id || !statuses || !n_deleted || !n_inserted ||
        !n_mutated || !pct_id || !pcts))) return C2B_E_ARG;
    FILE *fh = fopen(path, "wb");
    if (!fh) return C2B_E_ARG;
    static const char hdr[] = "Aligned_Sequence\tReference_Sequence\tReference_Name\tRead_Status\tn_deleted\tn_inserted\tn_mutated\t#Reads\t%Reads\n";
    bool ok = fwrite(hdr, 1, sizeof hdr - 1, fh) == sizeof hdr - 1;
    const int T = nthreads(n_threads, n_sel, 4096);
    const int64_t block = 1 << 16;                         // rows formatted per round and thread
    std::vector<std::string> bufs((size_t)T);
    for (int64_t base = 0; base < n_sel && ok; base += block * T) {
        parallel_for(T, [&](int t) {
            std::string &b = bufs[(size_t)t];
            b.clear();
            const int64_t lo = std::min(n_sel, base + block * t), hi = std::min(n_sel, lo + block);
            char num[64];
            for (int64_t k = lo; k < hi; k++) {
                const int64_t r = rows[k];
                const int n = A->len[(size_t)r];
                const char *p = (const char *)A->arena.data() + A->off[(size_t)r];
                b.append(p, (size_t)n); b.push_back('\t'); b.append(p + n, (size_t)n); b.push_back('\t');
                b.append(names[name_id[r]]); b.push_back('\t'); b.append(statuses[status_id[r]]); b.push_back('\t');
                const int m = snprintf(num, sizeof num, "%d\t%d\t%d\t%lld\t", n_deleted[r], n_inserted[r], n_mutated[r], (long long)A->count[(size_t)r]);
                b.append(num, (size_t)m);
                b.append(pcts[pct_id[r]]); b.push_back('\n');
            }
        });
        for (int t = 0; t < T && ok; t++) ok = fwrite(bufs[(size_t)t].data(), 1, bufs[(size_t)t].size(), fh) == bufs[(size_t)t].size();
    }
    ok = (fclose(fh) == 0) && ok;
    return ok ? C2B_OK : C2B_E_ARG;
}

}  // extern "C"

// pandas' group_sum for float64 (Kahan): one addend
static inline void group_add(double &sumx, double &comp, double val)
{
    const double y = val - comp;
    const double t = sumx + y;
    comp = t - sumx - y;
    if (comp != comp) comp = 0;                             // inf - inf
    sumx = t;
}

// pandas' groupby(six key columns).sum() over `rows` in row order (#Reads in int64, %Reads with group_add), then
// sort_values(['#Reads', 'Aligned_Sequence', 'Reference_Sequence'], ascending=[False, True, True]) from groupby's key order
std::vector<c2b_cut_group> c2b_group_around_cut(const std::vector<c2b_cut_group> &rows)
{
    std::vector<c2b_cut_group> groups;
    std::unordered_multimap<uint64_t, int64_t> index;
    index.reserve(std::min<size_t>(rows.size(), (size_t)1 << 20));
    for (const c2b_cut_group &R : rows) {
        uint64_t h = 1469598103934665603ull;
        auto mix = [&](uint64_t v) { h ^= v; h *= 1099511628211ull; };
        for (int64_t x = 0; x < R.len; x++) mix(R.seq[x]);
        mix(0x100);
        for (int64_t x = 0; x < R.len; x++) mix(R.ref[x]);
        mix(R.unedited ? 0x201 : 0x200); mix((uint64_t)R.ndel); mix((uint64_t)R.nins + 0x1000000ull); mix((uint64_t)R.nmut + 0x2000000ull);
        int64_t g = -1;
        auto range = index.equal_range(h);
        for (auto it = range.first; it != range.second; ++it) {
            const c2b_cut_group &G = groups[(size_t)it->second];
            if (G.len != R.len || G.unedited != R.unedited || G.ndel != R.ndel || G.nins != R.nins || G.nmut != R.nmut) continue;
            if (memcmp(G.seq, R.seq, (size_t)R.len) || memcmp(G.ref, R.ref, (size_t)R.len)) continue;
            g = it->second; break;
        }
        if (g < 0) {
            c2b_cut_group G = R;
            G.reads = 0; G.pct = 0.0; G.comp = 0.0;
            g = (int64_t)groups.size();
            groups.push_back(G);
            index.emplace(h, g);
        }
        c2b_cut_group &G = groups[(size_t)g];
        G.reads += R.reads;
        group_add(G.pct, G.comp, R.pct);
    }
    // groupby order (keys ascending) refined by the final sort_values(#Reads desc, Aligned_Sequence, Reference_Sequence), stable
    auto scmp = [](const uint8_t *pa, int64_t la, const uint8_t *pb, int64_t lb) {
        const int c = memcmp(pa, pb, (size_t)std::min(la, lb));
        if (c) return c;
        return la < lb ? -1 : la > lb ? 1 : 0;
    };
    std::sort(groups.begin(), groups.end(), [&](const c2b_cut_group &a, const c2b_cut_group &b) {
        if (a.reads != b.reads) return a.reads > b.reads;
        int c = scmp(a.seq, a.len, b.seq, b.len); if (c) return c < 0;
        c = scmp(a.ref, a.len, b.ref, b.len); if (c) return c < 0;
        if (a.unedited != b.unedited) return a.unedited < b.unedited;
        if (a.ndel != b.ndel) return a.ndel < b.ndel;
        if (a.nins != b.nins) return a.nins < b.nins;
        return a.nmut < b.nmut;
    });
    return groups;
}

extern "C" {

// get_dataframe_around_cut_asymmetrical over the rows `rows` (in the DataFrame's row order).  Returns the number of groups
// (< 0: error); fetch them with c2b_alleles_cut_fetch.  C2B_E_LIMIT: some row's alignment does not hold reference position
// cut_point (list.index raises ValueError in the reference).
int64_t c2b_alleles_around_cut(c2b_alleles *A, int64_t n_sel, const int64_t *rows, int32_t cut_point, int32_t plot_left, int32_t plot_right,
                               const uint8_t *unedited, const int32_t *n_deleted, const int32_t *n_inserted, const int32_t *n_mutated,
                               const double *pct)
{
    if (!A || n_sel < 0 || (n_sel && (!rows || !unedited || !n_deleted || !n_inserted || !n_mutated || !pct)) || cut_point < 0) return C2B_E_ARG;
    A->groups.clear();
    A->win_max = 0;
    auto window_of = [&](int64_t r, int &s0, int &s1) -> bool {
        const int n = A->len[(size_t)r];
        const uint8_t *rf = A->arena.data() + A->off[(size_t)r] + n;
        int seen = -1, c = 0;
        for (; c < n; c++) if (rf[c] != '-' && ++seen == cut_point) break;
        if (c == n) return false;
        long a = (long)c - plot_left + 1, b = (long)c + plot_right + 1;        // Python slice semantics
        if (a < 0) { a += n; if (a < 0) a = 0; }
        if (b < 0) { b += n; if (b < 0) b = 0; }
        if (a > n) a = n;
        if (b > n) b = n;
        if (b < a) b = a;
        s0 = (int)a; s1 = (int)b;
        return true;
    };
    std::vector<c2b_cut_group> cut((size_t)n_sel);
    for (int64_t k = 0; k < n_sel; k++) {
        const int64_t r = rows[k];
        if (r < 0 || r >= A->n) return C2B_E_ARG;
        int s0, s1;
        if (!window_of(r, s0, s1)) return C2B_E_LIMIT;
        const uint8_t *p = A->arena.data() + A->off[(size_t)r];
        c2b_cut_group &G = cut[(size_t)k];
        G.seq = p + s0; G.ref = p + A->len[(size_t)r] + s0; G.len = s1 - s0;
        G.unedited = unedited[r] ? 1 : 0; G.ndel = n_deleted[r]; G.nins = n_inserted[r]; G.nmut = n_mutated[r];
        G.reads = A->count[(size_t)r]; G.pct = pct[r];
    }
    A->groups = c2b_group_around_cut(cut);
    for (const c2b_cut_group &G : A->groups) if (G.len > A->win_max) A->win_max = (int32_t)G.len;
    return (int64_t)A->groups.size();
}

int32_t c2b_alleles_cut_width(const c2b_alleles *A) { return A ? A->win_max : 0; }

// seq / ref: n_groups * width bytes (width = c2b_alleles_cut_width()), each window left-justified; wlen its length
int c2b_alleles_cut_fetch(const c2b_alleles *A, uint8_t *seq, uint8_t *ref, int32_t *wlen, uint8_t *unedited, int32_t *n_deleted,
                          int32_t *n_inserted, int32_t *n_mutated, int64_t *reads, double *pct)
{
    if (!A || !seq || !ref || !wlen || !unedited || !n_deleted || !n_inserted || !n_mutated || !reads || !pct) return C2B_E_ARG;
    const int W = A->win_max;
    for (size_t g = 0; g < A->groups.size(); g++) {
        const c2b_cut_group &G = A->groups[g];
        memcpy(seq + g * (size_t)W, G.seq, (size_t)G.len);
        memcpy(ref + g * (size_t)W, G.ref, (size_t)G.len);
        wlen[g] = (int32_t)G.len; unedited[g] = G.unedited; n_deleted[g] = (int32_t)G.ndel; n_inserted[g] = (int32_t)G.nins;
        n_mutated[g] = (int32_t)G.nmut; reads[g] = G.reads; pct[g] = G.pct;
    }
    return C2B_OK;
}

}  // extern "C"
