// c2b_vcf.cuh -- the biallelic edit records of --vcf_output, built on the device from the packed detailed allele rows.
//
// Replaces the per-row work of build_edit_counts (CRISPResso2/writers/vcf.py:172-212): for every edited row, its deletions
// (_edits_from_deletions / _left_normalize_deletion, :9-76), its insertions (_edits_from_insertions /
// _left_normalize_insertion, :79-153) and its substitutions (_edits_from_substitutions, :156-169) become records
//   chrom id (int32) | VCF position (int64) | len(REF) (int32) | REF bytes | ALT bytes
// in the row's own order.  Equal records are summed on the host (c2b_vcf_sum_records in c2b_fastq.cpp).
//
// One warp per row.  Every ref_positions.index(p) is a ballot search for the first column holding p; control flow is
// warp-uniform, lane 0 stores the scalar fields, the lanes share byte copies.  The same routine runs twice: with no output
// buffer it counts records and bytes and notes the row's first Python exception (size pass), then, after a scan of the sizes,
// it writes (write pass).  Python's semantics are kept where hand-built rows can reach them: first match of index(), the
// ValueError fallback to index(end - 1), slice clamping and negative-start wrap, IndexError on a string index past the end or
// on the last character of an empty string, and max() over no non-negative position when the insertion generator starts.
//
// Compiled by nvcc for sm_90a (c2b_engine.cu) and by g++ against the warp emulator (tests/emu/): nothing here needs CUB.
#pragma once

namespace c2b {
namespace vcf {

// the first Python exception of a row (C2B_VCF_E_* of include/c2b200.h)
enum { E_NONE = 0, E_KEY = 1, E_NOT_IN_LIST = 2, E_STRING_INDEX = 3, E_EMPTY_MAX = 4 };

struct VParams {
    int64_t n;                                                 // rows of this chunk
    const int32_t *chrom; const int64_t *pos; const int64_t *reads;   // per row; chrom < 0: Reference_Name not in amplicon_positions
    const uint8_t *ref; const int64_t *ref_off;                // Reference_Sequence
    const uint8_t *aln; const int64_t *aln_off;                // Aligned_Sequence
    const int64_t *rp; const int64_t *rp_off;                  // ref_positions
    const int64_t *del; const int64_t *del_off;                // deletion_coordinates: (start, end) pairs, offsets in pairs
    const int64_t *ins; const int64_t *ins_off;                // insertion_coordinates: (left, right) pairs, offsets in pairs
    const int64_t *isz; const int64_t *isz_off;                // insertion_sizes
    const int64_t *sub; const int64_t *sub_off;                // substitution_positions
    int64_t *nrec, *nbytes, *err;                              // size pass: per row; err: [n][2] = kind, value
    const int64_t *rec_base, *key_off;                         // write pass: exclusive scans of nrec / nbytes (n + 1)
    uint8_t *keys; int64_t *rec_pos, *rec_w;                   // write pass: record bytes, each record's offset and #Reads
};

struct Row {
    const uint8_t *ref, *aln; int64_t RS, AS;
    const int64_t *rp; int64_t L;
};

// ref_positions.index(p): the first column holding p, -1 if none
C2B_DEV int64_t find(const Row &w, int64_t p)
{
    for (int64_t b = 0; b < w.L; b += 32) {
        const int64_t i = b + wp::lane();
        const uint32_t m = wp::ballot(i < w.L && w.rp[i] == p);
        if (m) return b + wp::ffs(m) - 1;
    }
    return -1;
}

// Python's s[a:b] on a string of length n -> [lo, hi)
C2B_DEV void py_slice(int64_t a, int64_t b, int64_t n, int64_t &lo, int64_t &hi)
{
    lo = a < 0 ? (a + n < 0 ? 0 : a + n) : (a > n ? n : a);
    hi = b < 0 ? (b + n < 0 ? 0 : b + n) : (b > n ? n : b);
    if (hi < lo) hi = lo;
}

struct Out {
    uint8_t *p; int64_t n;                                     // this row's key bytes (nullptr in the size pass)
    int64_t *pos, *w; int64_t rec, reads;                      // record offsets / weights from this row's first record on
    int64_t base;                                              // offset of this row's keys in the chunk's arena
};

C2B_DEV void put_le(Out &o, uint64_t v, int nb)
{
    if (o.p && wp::lane() < nb) o.p[o.n + wp::lane()] = (uint8_t)(v >> (8 * wp::lane()));
    o.n += nb;
}

// one record: header, then REF = a[0..na) and ALT = b0 (one byte) followed by the cyclic rotation of c[0..nc) right by k
C2B_DEV void record(Out &o, int32_t chrom, int64_t vpos, const uint8_t *a, int64_t na, uint8_t b0, bool has_b0, const uint8_t *c,
                    int64_t nc, int64_t k)
{
    if (o.p && wp::lane() == 0) { o.pos[o.rec] = o.base + o.n; o.w[o.rec] = o.reads; }
    o.rec++;
    put_le(o, (uint32_t)chrom, 4);
    put_le(o, (uint64_t)vpos, 8);
    put_le(o, (uint64_t)na, 4);
    if (o.p) for (int64_t i = wp::lane(); i < na; i += 32) o.p[o.n + i] = a[i];
    o.n += na;
    if (has_b0) { if (o.p && wp::lane() == 0) o.p[o.n] = b0; o.n++; }
    if (o.p && nc) {
        const int64_t s = k % nc;
        for (int64_t i = wp::lane(); i < nc; i += 32) o.p[o.n + i] = c[(i - s + nc) % nc];
    }
    o.n += nc;
}

// the row's records in the reference's order; -> E_NONE or the first exception (kind, value: the missing index() argument)
C2B_DEV int row_edits(const VParams &P, int64_t r, Out &o, int64_t &val)
{
    const int32_t chrom = P.chrom[r];
    if (chrom < 0) return E_KEY;                               // amplicon_positions[ref_name] (:203)
    const int64_t pos = P.pos[r];
    Row w;
    w.ref = P.ref + P.ref_off[r]; w.RS = P.ref_off[r + 1] - P.ref_off[r];
    w.aln = P.aln + P.aln_off[r]; w.AS = P.aln_off[r + 1] - P.aln_off[r];
    w.rp = P.rp + P.rp_off[r]; w.L = P.rp_off[r + 1] - P.rp_off[r];
#define C2B_VCF_INDEX(dst, p) do { const int64_t q_ = (p); (dst) = find(w, q_); if ((dst) < 0) { val = q_; return E_NOT_IN_LIST; } } while (0)
    // deletions (:43-76)
    for (int64_t d = P.del_off[r]; d < P.del_off[r + 1]; d++) {
        int64_t start = P.del[2 * d], end = P.del[2 * d + 1], ib, il;
        while (start > 0) {                                    // _left_normalize_deletion (:32-39)
            C2B_VCF_INDEX(ib, start - 1);
            C2B_VCF_INDEX(il, end - 1);
            if (ib >= w.RS || il >= w.RS) return E_STRING_INDEX;
            if (w.ref[ib] != w.ref[il]) break;
            start--; end--;
        }
        const int64_t left = start == 0 ? pos : pos + start - 1;
        int64_t rs, re;
        C2B_VCF_INDEX(rs, start);
        re = find(w, end);
        if (re < 0) C2B_VCF_INDEX(re, end - 1);                // the caught ValueError (:61-64)
        int64_t lo, hi;
        if (start == 0) {
            py_slice(rs, re + 1, w.RS, lo, hi);
            if (hi == lo) return E_STRING_INDEX;               // ref_seq[-1]
            record(o, chrom, left, w.ref + lo, hi - lo, w.ref[hi - 1], true, nullptr, 0, 0);
        } else {
            if (re == w.RS - 1) py_slice(rs - 1, re + 1, w.RS, lo, hi);
            else py_slice(rs - 1, re, w.RS, lo, hi);
            if (hi == lo) return E_STRING_INDEX;               // ref_seq[0]
            record(o, chrom, left, w.ref + lo, hi - lo, w.ref[lo], true, nullptr, 0, 0);
        }
    }
    // insertions (:115-153): max() over the non-negative positions runs when the generator starts
    int64_t ref_len = -1;
    for (int64_t b = 0; b < w.L; b += 32) {
        const int64_t i = b + wp::lane();
        int64_t v = (i < w.L && w.rp[i] >= 0) ? w.rp[i] : -1;
        for (int s = 16; s; s >>= 1) {                         // 64-bit max through two 32-bit shuffles
            const uint32_t lo = wp::shflu((uint32_t)(uint64_t)v, wp::lane() ^ s), hi = wp::shflu((uint32_t)((uint64_t)v >> 32), wp::lane() ^ s);
            const int64_t u = (int64_t)(((uint64_t)hi << 32) | lo);
            if (u > v) v = u;
        }
        if (v > ref_len) ref_len = v;
    }
    if (ref_len < 0) return E_EMPTY_MAX;
    ref_len += 1;
    const int64_t ni = P.ins_off[r + 1] - P.ins_off[r], ns = P.isz_off[r + 1] - P.isz_off[r];
    for (int64_t i = 0; i < ni; i++) {
        const int64_t la = P.ins[2 * (P.ins_off[r] + i)], ra = P.ins[2 * (P.ins_off[r] + i) + 1];
        const int64_t size = i < ns ? P.isz[P.isz_off[r] + i] : 0;
        int64_t rai, lo, hi;
        C2B_VCF_INDEX(rai, ra);
        py_slice(rai - size, rai, w.AS, lo, hi);               // ins_bases = aln_str[right_anchor_idx - size:right_anchor_idx]
        const int64_t nb = hi - lo;
        int64_t anchor = (la == ref_len && ref_len > 0) ? ref_len - 1 : la;
        int64_t k = 0;                                         // _left_normalize_insertion (:105-111): each step rotates ins_bases right
        while (anchor > 0) {
            int64_t ai;
            C2B_VCF_INDEX(ai, anchor);
            if (nb == 0) return E_STRING_INDEX;                // ins_bases[-1]
            if (ai >= w.RS) return E_STRING_INDEX;
            const uint8_t last = w.aln[lo + ((nb - 1 - k % nb) + nb) % nb];
            if (last != w.ref[ai]) break;
            anchor--; k++;
        }
        int64_t ci;
        C2B_VCF_INDEX(ci, anchor);
        if (ci >= w.RS) return E_STRING_INDEX;
        record(o, chrom, pos + anchor, w.ref + ci, 1, w.ref[ci], true, w.aln + lo, nb, k);
    }
    // substitutions (:156-169)
    for (int64_t s = P.sub_off[r]; s < P.sub_off[r + 1]; s++) {
        const int64_t sp = P.sub[s];
        int64_t ci;
        C2B_VCF_INDEX(ci, sp);
        if (ci >= w.RS || ci >= w.AS) return E_STRING_INDEX;
        record(o, chrom, pos + sp, w.ref + ci, 1, w.aln[ci], true, nullptr, 0, 0);
    }
#undef C2B_VCF_INDEX
    return E_NONE;
}

template <bool WRITE>
C2B_DEV void edits_one(const VParams &P, int64_t r)
{
    Out o;
    o.p = WRITE ? P.keys + P.key_off[r] : nullptr; o.n = 0;
    o.pos = WRITE ? P.rec_pos + P.rec_base[r] : nullptr; o.w = WRITE ? P.rec_w + P.rec_base[r] : nullptr;
    o.rec = 0; o.reads = P.reads[r]; o.base = WRITE ? P.key_off[r] : 0;
    int64_t val = 0;
    const int kind = row_edits(P, r, o, val);
    if (!WRITE && wp::lane() == 0) { P.nrec[r] = o.rec; P.nbytes[r] = o.n; P.err[2 * r] = kind; P.err[2 * r + 1] = val; }
}

// the first row with an exception -> first[0..2] = row, kind, value (row -1: none); one warp
C2B_DEV void first_error(const int64_t *err, int64_t n, int64_t *first)
{
    const int l = wp::lane();
    const int64_t seg = (n + 31) / 32, a = l * seg < n ? l * seg : n, b = a + seg < n ? a + seg : n;
    int64_t f = -1;
    for (int64_t i = a; i < b; i++) if (err[2 * i]) { f = i; break; }
    const uint32_t m = wp::ballot(f >= 0);
    if (l == 0) { first[0] = -1; first[1] = 0; first[2] = 0; }
    if (m && l == wp::ffs(m) - 1) { first[0] = f; first[1] = err[2 * f]; first[2] = err[2 * f + 1]; }
}

}  // namespace vcf
}  // namespace c2b

#ifndef C2B_EMU
__global__ void __launch_bounds__(256) c2b_vcf_size_kernel(const __grid_constant__ c2b::vcf::VParams P)
{
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < P.n; r += nw) c2b::vcf::edits_one<false>(P, r);
}
__global__ void __launch_bounds__(256, 1) c2b_vcf_write_kernel(const __grid_constant__ c2b::vcf::VParams P)
{
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < P.n; r += nw) c2b::vcf::edits_one<true>(P, r);
}
// exclusive scans of the record counts and key bytes (c2b::ann::scan_sizes), and the chunk's first exception
__global__ void __launch_bounds__(32) c2b_vcf_scan_kernel(const int64_t *nrec, int64_t *rec_base, const int64_t *nbytes, int64_t *key_off,
                                                         const int64_t *err, int64_t *first, int64_t n)
{
    c2b::ann::scan_sizes(nrec, rec_base, n);
    c2b::ann::scan_sizes(nbytes, key_off, n);
    c2b::vcf::first_error(err, n, first);
}
#endif
