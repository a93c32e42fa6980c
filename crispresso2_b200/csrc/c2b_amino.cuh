// c2b_amino.cuh -- the --coding_seq amino-acid allele table on the device: the per-row translation and the protein alignment.
//
// Replaces the per-row Python of get_amino_acid_row (CRISPResso2/CRISPRessoShared.py:1557-1623):
//   * row pass (codons_one): left_idx = row['ref_positions'].index(plot_left_idx) as a ballot search, then the gap-stripped
//     suffixes Aligned_Sequence[left_idx:] and Reference_Sequence[left_idx:] translated codon by codon
//     (get_amino_acids_and_codons, :478-484; a trailing 1-2 nt remainder is dropped).  Per row: the read and reference protein
//     strings and each residue's codon index (16 a + 4 b + c over A C G T), or the row's failure: plot_left_idx missing
//     (ValueError), a codon outside the table (KeyError; the read is translated first), or a translation shorter than one codon
//     (the reference's global_align is undefined on an empty string).
//   * protein alignment (protein_one): CRISPResso2Align.global_align (Align.pyx:101-434) of one read protein against one
//     reference protein, forward strand, no seed test, with the general kernel's own 32-bit DP and traceback (align_strand:
//     dp_block over row blocks, walk_batch).  Those blocks index the substitution profile by read code and never read the
//     alphabet size, so a profile of up to 32 read codes needs no change to them.  The packed 16-bit path, the ring and the
//     diagonal tier are never entered: they classify DNA reads, and the packed path's admission (min score + 2 beta >= 0)
//     refuses BLOSUM62 at -1/-1 anyway.
// Silent edits, truncation and the grouping are on the host (c2b_amino_table in c2b_engine.cu).
//
// Compiled by nvcc for sm_90a (c2b_engine.cu) and by g++ against the warp emulator (tests/emu/).
#pragma once

namespace c2b {
namespace aa {

// a row's failure (C2B_AA_E_* of include/c2b200.h)
enum { E_NONE = 0, E_NOT_IN_LIST = 1, E_CODON = 2, E_EMPTY = 3, E_UNDEFINED = 4 };   // E_UNDEFINED: set by the host

struct RParams {
    int64_t n;                                                 // rows of this chunk
    int64_t left;                                              // plot_left_idx
    const uint8_t *ref; const int64_t *ref_off;                // Reference_Sequence
    const uint8_t *aln; const int64_t *aln_off;                // Aligned_Sequence
    const int64_t *rp; const int64_t *rp_off;                  // ref_positions
    const uint8_t *table;                                      // [64] codon index -> amino acid
    uint8_t *raa, *rcod;                                       // read protein / codon indices at aln_off[r] (room: len(Aligned_Sequence))
    uint8_t *faa, *fcod;                                       // reference protein / codon indices at ref_off[r]
    int64_t *len;                                              // [n][2]: read residues, reference residues
    int64_t *err;                                              // [n]: E_*
};

C2B_DEV int nt_code(uint8_t c) { return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1; }

// s[from:].replace('-', '') translated: the nucleotides are first compacted into cod[] (room: len(s)), then codon k is read
// from cod[3k..3k+2] and its index written back to cod[k] -- all lanes read a batch of 32 codons before any writes, and a
// batch's writes (cod[32 i ..]) lie below every later batch's reads (cod[96 i ..]).  -> residues, or -1 on a codon outside the
// table (KeyError)
C2B_DEV int64_t translate(const uint8_t *s, int64_t from, int64_t len, const uint8_t *table, uint8_t *aa, uint8_t *cod)
{
    const uint32_t below = (1u << wp::lane()) - 1u;
    int64_t k = 0;
    for (int64_t b = from; b < len; b += 32) {
        const int64_t i = b + wp::lane();
        const bool base = i < len && s[i] != '-';
        const uint32_t m = wp::ballot(base);
        if (base) cod[k + wp::popc(m & below)] = s[i];
        k += wp::popc(m);
    }
    wp::sync();
    const int64_t nc = k / 3;
    bool bad = false;
    for (int64_t b = 0; b < nc; b += 32) {
        const int64_t c = b + wp::lane();
        int idx = 0;
        if (c < nc) {
            const int x = nt_code(cod[3 * c]), y = nt_code(cod[3 * c + 1]), z = nt_code(cod[3 * c + 2]);
            if (x < 0 || y < 0 || z < 0) bad = true;
            else idx = 16 * x + 4 * y + z;
        }
        wp::sync();
        if (c < nc) { cod[c] = (uint8_t)idx; aa[c] = table[idx]; }
        wp::sync();
    }
    return wp::ballot(bad) ? -1 : nc;
}

C2B_DEV void codons_one(const RParams &P, int64_t r)
{
    const int64_t *rp = P.rp + P.rp_off[r];
    const int64_t np = P.rp_off[r + 1] - P.rp_off[r];
    int64_t left = -1;                                         // first column whose ref_positions value is plot_left_idx
    for (int64_t b = 0; b < np && left < 0; b += 32) {
        const int64_t i = b + wp::lane();
        const uint32_t m = wp::ballot(i < np && rp[i] == P.left);
        if (m) left = b + wp::ffs(m) - 1;
    }
    int kind = E_NONE;
    int64_t na = 0, nf = 0;
    if (left < 0) kind = E_NOT_IN_LIST;
    else {
        const int64_t a0 = P.aln_off[r], f0 = P.ref_off[r];
        na = translate(P.aln + a0, left, P.aln_off[r + 1] - a0, P.table, P.raa + a0, P.rcod + a0);
        if (na < 0) kind = E_CODON;
        else {
            nf = translate(P.ref + f0, left, P.ref_off[r + 1] - f0, P.table, P.faa + f0, P.fcod + f0);
            kind = nf < 0 ? E_CODON : (na == 0 || nf == 0) ? E_EMPTY : E_NONE;
        }
    }
    if (wp::lane() == 0) { P.len[2 * r] = na; P.len[2 * r + 1] = nf; P.err[r] = kind; }
}

struct PParams {
    KParams K;                                                 // go, ge, TS; tb / bnd: per-warp slabs of the DP and its boundary rows
    RefDev R;                                                  // the reference protein: I, row blocks, prof [nq][Ipad], cIe, g4
    const uint8_t *codes; const int64_t *off; int64_t n;       // read proteins as alphabet codes
    uint64_t *ops;                                             // [n][32]: op stream (lane L: columns 32L.. from the right)
    int32_t *nops;                                             // [n]: alignment columns, or -1 when the walk failed
};

// global_align of read r on warp slot w
C2B_DEV void protein_one(const PParams &P, int64_t r, int64_t w)
{
    const int J = (int)(P.off[r + 1] - P.off[r]);
    const Walked wk = align_strand(P.K, P.R, P.codes + P.off[r], J, P.K.tb + w * P.K.tb_words_per_warp,
                                   P.K.bnd + w * P.K.bnd_words_per_warp);
    P.ops[r * 32 + wp::lane()] = wk.ops;
    if (wp::lane() == 0) P.nops[r] = wk.err ? -1 : wk.n;
}

}  // namespace aa
}  // namespace c2b

#ifndef C2B_EMU
__global__ void __launch_bounds__(256) c2b_amino_codons_kernel(const __grid_constant__ c2b::aa::RParams P)
{
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < P.n; r += nw) c2b::aa::codons_one(P, r);
}
// one read per warp; warp slot w owns slab w (the grid has at most as many warps as the slabs)
__global__ void __launch_bounds__(256) c2b_protein_kernel(const __grid_constant__ c2b::aa::PParams P)
{
    const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = w; r < P.n; r += nw) c2b::aa::protein_one(P, r, w);
}
#endif
