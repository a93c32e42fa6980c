// c2b_base_edit.cuh -- the per-row work of the --base_editor_output allele tables, on the device from packed allele rows.
//
// Replaces the per-row Python of
//   * get_upset_plot_counts (CRISPResso2/plots/data_prep.py:1869-1988; its copy CRISPRessoCORE.py:209-327) and
//     get_refpos_values (data_prep.py:1816-1856): for every row on the wild-type reference, the read bases that belong to each
//     target position, their category (R, T, D, I, N, first match wins, :1923-1938) and the binary / category / precise keys
//     ("\t"-joined fields + "\t" + str(has_indel), :1958-1960).  Each key becomes one record
//       tag (0 binary, 1 category, 2 precise) | key text
//     weighted by the row's #Reads; equal records are summed on the host (c2b_vcf_sum_records) and the category codes give the
//     per-position counts and the totals (c2b_be_upset_counts in c2b_engine.cu).
//   * get_base_edit_row_around_cut (CRISPRessoShared.py:1472-1488): the Aligned_Sequence characters at the columns where
//     Reference_Sequence holds conversion_nuc_from.  Grouping and sorting are on the host (c2b_group_around_cut).
//
// One warp per row; the lanes walk the alignment 32 columns at a time.  Reference position k of get_refpos_values is the k-th
// non-gap reference column c_k (a ballot of the non-gap columns with a popcount prefix); its read bases are the columns
// [c_k, c_{k+1}) (gap columns go to the last non-gap position before them), position 0 starts at column 0 (a leading gap run
// goes to it), and the last position runs to the end of the reference string.  An all-gap reference gives position 0 the
// read's first len(Reference_Sequence) characters.  Any other position is '' (the defaultdict(str) miss).
//
// Compiled by nvcc for sm_90a (c2b_engine.cu) and by g++ against the warp emulator (tests/emu/): nothing here needs CUB.
#pragma once

namespace c2b {
namespace be {

// the row's Python exception (C2B_BE_E_* of include/c2b200.h)
enum { E_NONE = 0, E_STRING_INDEX = 1 };
// categories of a target position (C2B_BE_CAT_*), in the order they are tested
enum { CAT_R = 0, CAT_T = 1, CAT_D = 2, CAT_I = 3, CAT_N = 4 };

struct UParams {
    int64_t n;                                                 // rows of this chunk
    const uint8_t *flags;                                      // per row: bit 0 Reference_Name == wt_ref_name, bit 1 has_indel
    const int64_t *reads;                                      // #Reads
    const uint8_t *ref; const int64_t *ref_off;                // Reference_Sequence
    const uint8_t *aln; const int64_t *aln_off;                // Aligned_Sequence
    int32_t nt;                                                // targets (entries of bp_substitutions_arr)
    const int64_t *tpos;                                       // target t: reference position, ref_base at tstr[toff[2t] ..
    const uint8_t *tstr; const int64_t *toff;                  //   toff[2t+1]), mod_base at tstr[toff[2t+1] .. toff[2t+2])
    int64_t *nrec, *nbytes, *err;                              // size pass: per row; err: [n][2] = kind, 0
    const int64_t *rec_base, *key_off;                         // write pass: exclusive scans of nrec / nbytes (n + 1)
    uint8_t *keys; int64_t *rec_pos, *rec_w;                   // write pass: record bytes, each record's offset and #Reads
    uint8_t *codes;                                            // write pass: codes[r * nt + t] = CAT_* (rows on wt_ref_name)
};

struct Row {
    const uint8_t *ref, *aln; int64_t RS;
};

// columns of the k-th and (k+1)-th non-gap reference characters (k >= 0); RS where the reference has fewer
C2B_DEV void base_cols(const Row &w, int64_t k, int64_t &ck, int64_t &ck1)
{
    ck = ck1 = w.RS;
    int64_t seen = 0;
    const uint32_t below = (1u << wp::lane()) - 1u;
    for (int64_t b = 0; b < w.RS; b += 32) {
        const int64_t i = b + wp::lane();
        const bool base = i < w.RS && w.ref[i] != '-';
        const uint32_t m = wp::ballot(base);
        const int64_t rank = seen + wp::popc(m & below);
        const uint32_t h0 = wp::ballot(base && rank == k), h1 = wp::ballot(base && rank == k + 1);
        if (h0) ck = b + wp::ffs(h0) - 1;
        if (h1) { ck1 = b + wp::ffs(h1) - 1; return; }
        seen += wp::popc(m);
    }
}

// the read bases of reference position p: aln[s .. e) (s == e: '')
C2B_DEV void segment(const Row &w, int64_t p, int64_t &s, int64_t &e)
{
    s = e = 0;
    if (p < 0) return;
    int64_t ck, ck1;
    base_cols(w, p, ck, ck1);
    if (p == 0) { s = 0; e = ck1; return; }                    // leading gap run and position 0 (all gaps: the whole string)
    if (ck == w.RS) return;                                    // past the last reference base
    s = ck; e = ck1;
}

// a[0..na) == b[0..nb)
C2B_DEV bool equal(const uint8_t *a, int64_t na, const uint8_t *b, int64_t nb)
{
    if (na != nb) return false;
    for (int64_t i = 0; i < na; i += 32) {
        const int64_t j = i + wp::lane();
        if (wp::ballot(j < na && a[j] != b[j])) return false;
    }
    return true;
}

// the row's three records; with WRITE the bytes, record offsets / weights and category codes, else the sizes and the error
template <bool WRITE>
C2B_DEV void upset_one(const UParams &P, int64_t r)
{
    const uint8_t f = P.flags[r];
    Row w;
    w.ref = P.ref + P.ref_off[r]; w.RS = P.ref_off[r + 1] - P.ref_off[r];
    w.aln = P.aln + P.aln_off[r];
    const int64_t AS = P.aln_off[r + 1] - P.aln_off[r];
    const bool on_ref = f & 1, indel = f & 2;
    // ref_aln_seq[0] of an empty string, or read_aln_seq[i] for some i < len(ref_aln_seq) (:1835-1849)
    const int kind = on_ref && (w.RS == 0 || AS < w.RS) ? E_STRING_INDEX : E_NONE;
    if (!on_ref || kind) {
        if (!WRITE && wp::lane() == 0) { P.nrec[r] = 0; P.nbytes[r] = 0; P.err[2 * r] = kind; P.err[2 * r + 1] = 0; }
        return;
    }
    const int nt = P.nt, tabs = nt > 0 ? nt : 1, nb = indel ? 4 : 5;
    const int64_t K1 = 1 + nt + tabs + nb;                     // tag + binary (or category) key
    uint8_t *o = WRITE ? P.keys + P.key_off[r] : nullptr;
    int64_t pos = 2 * K1 + 1;                                  // write position in the precise record
    for (int t = 0; t < nt; t++) {
        int64_t s, e;
        segment(w, P.tpos[t], s, e);
        const uint8_t *rb = P.tstr + P.toff[2 * t], *mb = P.tstr + P.toff[2 * t + 1];
        const int64_t nr = P.toff[2 * t + 1] - P.toff[2 * t], nm = P.toff[2 * t + 2] - P.toff[2 * t + 1], n = e - s;
        int cat;
        if (equal(w.aln + s, n, rb, nr)) cat = CAT_R;
        else if (equal(w.aln + s, n, mb, nm)) cat = CAT_T;
        else if (n == 1 && w.aln[s] == '-') cat = CAT_D;
        else if (n != 1) cat = CAT_I;
        else cat = CAT_N;
        if (WRITE) {
            for (int64_t i = wp::lane(); i < n; i += 32) o[pos + i] = w.aln[s + i];
            if (wp::lane() == 0) {
                o[1 + 2 * t] = cat == CAT_T ? 'T' : 'X';
                o[K1 + 1 + 2 * t] = "RTDIN"[cat];
                if (t + 1 < nt) { o[2 + 2 * t] = '\t'; o[K1 + 2 + 2 * t] = '\t'; o[pos + n] = '\t'; }
                P.codes[r * nt + t] = (uint8_t)cat;
            }
        }
        pos += n + (t + 1 < nt ? 1 : 0);
    }
    if (WRITE) {
        if (wp::lane() == 0) {
            const char *b = indel ? "True" : "False";
            const int64_t at[3] = {0, K1, 2 * K1};
            const int64_t tail[3] = {K1 - nb - 1, 2 * K1 - nb - 1, pos};   // the "\t" + str(has_indel) of each key
            for (int k = 0; k < 3; k++) {
                o[at[k]] = (uint8_t)k;
                o[tail[k]] = '\t';
                for (int i = 0; i < nb; i++) o[tail[k] + 1 + i] = (uint8_t)b[i];
                P.rec_pos[P.rec_base[r] + k] = P.key_off[r] + at[k];
                P.rec_w[P.rec_base[r] + k] = P.reads[r];
            }
        }
    } else if (wp::lane() == 0) {
        P.nrec[r] = 3; P.nbytes[r] = pos + 1 + nb; P.err[2 * r] = E_NONE; P.err[2 * r + 1] = 0;
    }
}

struct QParams {
    int64_t n;                                                 // rows of this chunk
    int32_t nuc;                                               // conversion_nuc_from, -1 when it is not one character
    const uint8_t *ref; const int64_t *ref_off;                // Reference_Sequence
    const uint8_t *aln; const int64_t *aln_off;                // Aligned_Sequence
    uint8_t *out;                                              // row r's projection at out[ref_off[r] ..]
    int64_t *len, *err;                                        // per row: projection length; 1: a column past the end of Aligned_Sequence
};

// [row['Aligned_Sequence'][i] for i in include_inds]: a ballot of Reference_Sequence == nuc, its popcount prefix places each
// selected character
C2B_DEV void quilt_one(const QParams &P, int64_t r)
{
    const uint8_t *ref = P.ref + P.ref_off[r], *aln = P.aln + P.aln_off[r];
    const int64_t RS = P.ref_off[r + 1] - P.ref_off[r], AS = P.aln_off[r + 1] - P.aln_off[r];
    uint8_t *o = P.out + P.ref_off[r];
    const uint32_t below = (1u << wp::lane()) - 1u;
    int64_t k = 0;
    bool bad = false;
    if (P.nuc >= 0)
        for (int64_t b = 0; b < RS; b += 32) {
            const int64_t i = b + wp::lane();
            const bool hit = i < RS && ref[i] == (uint8_t)P.nuc;
            const uint32_t m = wp::ballot(hit);
            if (hit && i < AS) o[k + wp::popc(m & below)] = aln[i];
            if (wp::ballot(hit && i >= AS)) bad = true;
            k += wp::popc(m);
        }
    if (wp::lane() == 0) { P.len[r] = k; P.err[r] = bad ? 1 : 0; }
}

}  // namespace be
}  // namespace c2b

#ifndef C2B_EMU
__global__ void __launch_bounds__(256) c2b_be_upset_size_kernel(const __grid_constant__ c2b::be::UParams P)
{
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < P.n; r += nw) c2b::be::upset_one<false>(P, r);
}
__global__ void __launch_bounds__(256) c2b_be_upset_write_kernel(const __grid_constant__ c2b::be::UParams P)
{
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < P.n; r += nw) c2b::be::upset_one<true>(P, r);
}
__global__ void __launch_bounds__(256) c2b_be_quilt_kernel(const __grid_constant__ c2b::be::QParams P)
{
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < P.n; r += nw) c2b::be::quilt_one(P, r);
}
#endif
