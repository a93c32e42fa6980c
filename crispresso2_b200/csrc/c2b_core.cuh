// c2b_core.cuh -- warp-level align + traceback + classification for CRISPResso2's per-read hot path.
//
// One warp owns one read.  For every (read, reference, strand) it runs
//   1. dp_block<KSTAR>  : the three-state affine Needleman-Wunsch of CRISPResso2Align.global_align
//                         (reference: CRISPResso2/CRISPResso2Align.pyx:142-317) as an anti-diagonal
//                         wavefront -- lane l owns reference rows 8l+1..8l+8 and steps over read columns,
//                         lane edges travel by warp shuffle, 4 traceback bits per cell go to an
//                         L2-resident scratch slab (one coalesced 128-byte row per step);
//   2. walk             : the traceback of Align.pyx:338-421, warp-uniform, reading the slab through a
//                         32-column shuffle window, producing a 2-bit op stream held in registers;
//   3. columns          : lane-parallel emission of the aligned strings (right-aligned, 16-byte vector
//                         stores), match count, and a per-reference-position scatter into shared memory;
//   4. rows             : find_indels_substitutions (CRISPRessoCOREResources.pyx:68-187) + the per-read
//                         part of the quantification loop (CRISPRessoCORE.py:3964-4115) evaluated in
//                         reference-position space with ballots, emitting scalars, the edit list and the
//                         per-position count vectors (integer atomics).
//
// Exactness device: every DP value is stored as 4*score + tag with tag(M)=0 < tag(J)=1 < tag(I)=2, so that a
// plain integer max reproduces the reference's strict-'>' cascades (ties: I beats J beats M,
// Align.pyx:195-229) and the winner's identity is the low two bits of the max.
//
// The same header is compiled by nvcc for sm_90a (c2b_engine.cu) and by g++ against a fiber-based warp
// emulator (tests/emu/) -- the emulator exists only so the kernel logic can be checked on a CPU-only box.
#pragma once
#include <stdint.h>
#include "c2b200.h"

#ifndef C2B_EMU
#include <cuda_runtime.h>
#define C2B_DEV __device__ __forceinline__
#define C2B_DEVNOINL __device__ __noinline__
namespace wp {
C2B_DEV int lane() { return threadIdx.x & 31; }
C2B_DEV int shfl_up(int v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
C2B_DEV int shfl(int v, int src) { return __shfl_sync(0xffffffffu, v, src); }
C2B_DEV uint32_t shflu(uint32_t v, int src) { return __shfl_sync(0xffffffffu, v, src); }
C2B_DEV uint32_t shflu_up(uint32_t v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
C2B_DEV int shfl_xor(int v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
C2B_DEV uint32_t ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
C2B_DEV void sync() { __syncwarp(); }
// barrier among the g warps of this warp's phase set (g consecutive warps): named barrier 1 + set index.  Out of line: ONE
// barrier instruction in the binary, so every warp of a set waits at the same PC whatever path it is on
__device__ __noinline__ void grp_sync(int g)
{
    // g is a power of two: shifts, not the integer divisions that used to be inlined at every one of the dozen phase barriers
    const int w = (int)(threadIdx.x >> 5), sh = 31 - __clz(g);
    const int set = w >> sh;
    // barrier.sync without .aligned (bar.sync is the aligned form): a warp may arrive not fully converged
    asm volatile("barrier.sync %0, %1;" ::"r"(1 + set), "r"(32 << sh) : "memory");
}
C2B_DEV int max3(int a, int b, int c) { return __vimax3_s32(a, b, c); }
C2B_DEV int addmax(int a, int b, int c) { return __viaddmax_s32(a, b, c); }   // max(a+b, c)
C2B_DEV uint32_t max3_2(uint32_t a, uint32_t b, uint32_t c) { return __vimax3_s16x2(a, b, c); }      // per signed half
C2B_DEV uint32_t addmax_2(uint32_t a, uint32_t b, uint32_t c) { return __viaddmax_s16x2(a, b, c); }  // per half max(a+b, c)
C2B_DEV uint4 ldg4u(const uint4 *p) { return __ldg(p); }
C2B_DEV void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
C2B_DEV int grid_warps() { return (int)(gridDim.x * (blockDim.x >> 5)); }
// shared-state-space accesses through a 32-bit address kept in a register (no generic-address arithmetic in hot loops)
C2B_DEV uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
C2B_DEV uint32_t lds_u8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
// 16 bytes global -> shared that land in the background (cp.async); wait_async: every copy this thread issued has landed
C2B_DEV void cp_async16(void *dst, const void *src)
{ asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_addr(dst)), "l"(__cvta_generic_to_global(src)) : "memory"); }
C2B_DEV void wait_async() { asm volatile("cp.async.wait_all;" ::: "memory"); }
C2B_DEV uint4 lds_v4(uint32_t a) { uint4 v; asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a)); return v; }
C2B_DEV uint2 ldcg2(const uint2 *p) { return __ldcg(p); }
C2B_DEV uint32_t funnel_r(uint32_t lo, uint32_t hi, int sh) { return __funnelshift_r(lo, hi, sh); }   // (hi:lo) >> sh
C2B_DEV int popc(uint32_t x) { return __popc(x); }
C2B_DEV int popcll(uint64_t x) { return __popcll(x); }
C2B_DEV int clz(uint32_t x) { return __clz(x); }
C2B_DEV int ffs(uint32_t x) { return __ffs(x); }
C2B_DEV uint32_t ldcg(const uint32_t *p) { return __ldcg(p); }
C2B_DEV int ldcgi(const int *p) { return __ldcg(p); }
C2B_DEV uint64_t ldcg64(const uint64_t *p) { return __ldcg((const unsigned long long *)p); }
C2B_DEV int4 ldg4(const int4 *p) { return __ldg(p); }
// explicit state spaces: a generic-pointer atomicAdd expands into an address-space dispatch at every call site
C2B_DEV void addg(unsigned long long *p, long long v)
{ asm volatile("red.global.add.u64 [%0], %1;" ::"l"(__cvta_generic_to_global(p)), "l"((unsigned long long)v) : "memory"); }
C2B_DEV void maxg(unsigned long long *p, unsigned long long v)
{ asm volatile("red.global.max.u64 [%0], %1;" ::"l"(__cvta_generic_to_global(p)), "l"(v) : "memory"); }
C2B_DEV uint32_t adds(uint32_t *p, uint32_t v)
{ uint32_t o; asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(o) : "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(v) : "memory"); return o; }
C2B_DEV unsigned long long fetch_work(unsigned long long *p)
{ unsigned long long o; asm volatile("atom.global.add.u64 %0, [%1], %2;" : "=l"(o) : "l"(__cvta_generic_to_global(p)), "l"(1ull) : "memory"); return o; }
C2B_DEV unsigned long long fetch_add(unsigned long long *p, unsigned long long v)
{ unsigned long long o; asm volatile("atom.global.add.u64 %0, [%1], %2;" : "=l"(o) : "l"(__cvta_generic_to_global(p)), "l"(v) : "memory"); return o; }
}  // namespace wp

#else
#include "warp_emu.h"   // provides C2B_DEV, C2B_DEVNOINL, int4/uint4 and namespace wp
namespace wp {
C2B_DEV int grid_warps() { return 1; }                  // the emulator runs a kernel's loop as a grid of one warp
C2B_DEV void cp_async16(void *dst, const void *src) { memcpy(dst, src, 16); }
C2B_DEV void wait_async() {}
}  // namespace wp
#endif

namespace c2b {

constexpr int MAXJ = C2B_MAX_READ_LEN;
constexpr int MAXI = C2B_MAX_REF_LEN;
constexpr int OP_M = 0, OP_J = 1, OP_I = 2, OP_NONE = 3;   // = DP tags; J: gap in read (deletion), I: gap in ref

// Per-reference device tables (built on the host by c2b_configure; "Ipad" = rows padded to 256).
struct RefDev {
    int32_t I, nrb, kstar, lstar, Ipad;
    int32_t gi0_4;                 // 4*gap_incentive[0]
    int32_t nseeds, seed_len;
    double min_aln;
    const int32_t *prof;           // [nq][Ipad]  4*matrix[ref[row]][alphabet[q]]
    const int32_t *cIe;            // [Ipad]      4*(gap_extend + gi[row+1])
    const int32_t *g4;             // [Ipad]      4*gi[row]                 (incentive of the row above, "i-1")
    const uint8_t *asc;            // [Ipad]      reference ASCII
    const uint8_t *rcode;          // [Ipad]      reference base as alphabet code, 255 if not in alphabet
    const uint8_t *incl;           // [Ipad+1]    bit 0: inside the quantification window; bit 1: exon position; bit 2: splicing position
    const uint16_t *cum;           // [Ipad+2]    cum[p] = #window positions < p
    const uint16_t *cumx, *cums;   // [Ipad+2]    same prefix counts for exon / splicing positions (coding only)
    int32_t coding, tem, hist_zero;   // refs[..]['contains_coding_seq'], sum(exon_len_mods), bucket of key 0 in the frame histograms
    unsigned long long *hist;      // [C2B_NHIST][hstride]
    uint64_t fw_seed[C2B_MAX_SEEDS], rc_seed[C2B_MAX_SEEDS];   // 3 bits per base, first base lowest
    unsigned long long *vec;       // [C2B_NVEC][vstride]
    unsigned long long *scal;      // [C2B_NSCAL]
    // packed two-reads-per-warp path (16-bit halves, biased scores; DESIGN.md section 6)
    int32_t pk_maxJ;               // longest read for which the 16-bit path is proven exact for this reference (0: never)
    uint32_t pk_XB, pk_YB, pk_M00; // border constants: X[0][j], Y[i][0], M[0][0] in both halves
    const uint32_t *prof2;         // [nq*nq][nrb][2][32][4]: for base pair q2, row block rb, lane l: words l*4.. of half 0 are
                                   // rows 8l..8l+3, of half 1 rows 8l+4..8l+7; halves of a word: 4*(score+2*beta) of read A / B
    const uint32_t *cIe2;          // [Ipad]         4*gi[row+1] in both halves
    const uint32_t *g42;           // [Ipad]         4*gi[row]   in both halves
    // ring-banded path (four pairs per warp): score bound of any alignment that leaves the band, see ring_bound()
    int32_t rg_ok, rg_smax, rg_gmax, rg_gsum;
    // diagonal tier (c2b_diag_kernel, DESIGN.md section 3): a read with J == I whose ungapped score beats dg_thr4 and the exact
    // edge-run scores of the offsets 1..dg_S on either side is aligned on the main diagonal, no DP needed
    int32_t dg_ok, dg_S, dg_thr4;
    int32_t dg_c4[2 * 4 + 1];      // [s + 4]: 4 x (gap costs + incentives) of the path on offset diagonal s (edge runs only)
    // every amplicon base has a code in 0..3 and the scores it meets from codes 0..3 are two-valued: dg_a4 = 4 x the score of
    // the amplicon's own code, dg_b4 = 4 x that of any other; the tier then scores a read of codes 0..3 by popcounts
    int32_t dg_two, dg_a4, dg_b4;
    // routing of the tier's unproved reads (route_read, DESIGN.md section 3): a read whose lower bound on its best one-gap
    // path does not beat rt_thr (the narrow band's ring_bound at J == I) goes straight to the wide ring
    int32_t rt_ok, rt_thr;
    int32_t rt_mx;                 // least match score minus least other score (ACGT codes; everything else never matches)
    int32_t rt_c[32];              // [s + 16]: gap and edge-run costs of offset s + least score of its I - |s| diagonal columns
                                   // (RT_OFF: offset not tried -- s == 0, or outside the narrow band)
    const uint4 *rt_pl;            // [Ipad/32 + 2]: reference codes as bit planes (x: bit 0, y: bit 1, z: code in ACGT), zero past I
};
constexpr int32_t RT_OFF = -(1 << 30);
// the narrow first tier's band (align_narrow16): paths inside column - row in [-RN_DLO, RN_DHI] are computed exactly
constexpr int RN_DLO = 17, RN_DHI = 11;

// The engine's work block in device memory: what the kernels count for the host, and the hand-out counters and list lengths
// of the launch sequence in flight.
struct WorkBlock {
    // cumulative path statistics (c2b_path_counts): general kernel work items through the pair path and read by read, packed
    // pairs re-run over the full matrix; in reads: kept by the ring, sent on to the full matrix, settled by the ALIGN kernel
    unsigned long long pair_items, single_items, band_reruns, ring_kept, ring_sent, align_settled;
    // cumulative, the diagonal tier (c2b_diag_counts, c2b_route_counts): reads proved, put on its list, sent to the second tier
    // (routed there or failed by the narrow tier), routed, kept for the narrow tier
    unsigned long long diag_proved, diag_listed, tier2, routed, kept;
    unsigned long long diag_popc;          // cumulative (c2b_diag_popcount_reads): reads the diagonal tier scored by popcounts
    struct Launch {                        // zeroed at the start of every launch sequence
        // work hand-out counters: ALIGN (or the general kernel alone), the second-tier ALIGN launch, the general kernel after ALIGN
        unsigned long long align_next, tier2_next, general_next;
        unsigned long long widest;         // widest alignment of the batch (all kernels of the launch sequence)
        // list lengths: pairs left over for the general kernel, the tier-2 list, the narrow tier's and the diagonal tier's list
        unsigned long long left_n, tier2_n, narrow_n, diag_n;
    } launch;
};
constexpr size_t WORK_BYTES = 32 * 8;
static_assert(sizeof(WorkBlock) <= WORK_BYTES, "work block");

struct KParams {
    const uint8_t *reads; const int64_t *offsets; int64_t n_reads;
    const int32_t *count, *qweight, *ref_id;
    const int32_t *pair_order;        // optional: work item w handles reads pair_order[2w], pair_order[2w+1] (equal lengths adjacent)
    c2b_read_rec *recs; c2b_aln_rec *alns; uint8_t *strings; c2b_edit *edits;
    int32_t W, edit_cap;
    const RefDev *refs; int32_t n_refs;
    int32_t out_refs, ops_refs;       // output slots per read (1 when ref_id is given: compact Pooled layout, else n_refs); opsbuf refs per warp
    int32_t go, ge, seed_count, seed_min; uint32_t flags; int32_t nq;
    uint8_t alpha[C2B_MAX_Q]; uint8_t comp[C2B_MAX_Q];
    uint32_t *tb; int64_t tb_words_per_warp; int32_t TS;      // TS = steps stride per row block (maxJ + 32)
    uint32_t *tbb; int64_t tbb_words_per_warp;                // banded slab of the packed path (PK_BAND_SLOTS slots per lane)
    uint32_t *tbq;                                            // slab of the ring-banded path: [step][lane] uint2, TS steps per warp
    int32_t *bnd; int64_t bnd_words_per_warp;                 // 2 x 3 x (maxJ+1): row-block boundary rows
    uint64_t *opsbuf;                                         // [warp][n_refs][32] op streams (multi-reference)
    uint64_t *rgops;                                          // [warp][RG_MAX_REFS][4 pairs][RG_OPS_STRIDE]: walked op streams of the multi-reference ring path
    WorkBlock *wb;
    unsigned long long *work_counter;      // work hand-out counter of this launch (a field of wb->launch)
    // two-kernel form (c2b_split.cuh): op streams and their meta word per (read, reference) slot, written by the ALIGN kernel
    // (and by the general kernel for the pairs it aligns), read by the CLASSIFY kernel and copied out as the compact output
    uint64_t *gops; uint32_t *gmeta; int32_t NW;            // NW = W / 32 words of 32 ops per slot
    int32_t *left;                                          // ALIGN kernel: pairs left over for the general kernel (wb->launch.left_n)
    int32_t *left2;                                         // ALIGN kernel, narrow first tier: reads for the second-tier launch (nullptr: no narrow tier)
    int32_t *left0;                                         // diagonal tier: reads it did not prove (CLASSIFY's list)
    int32_t *left1;                                         // diagonal tier with routing: the unproved reads it keeps for the narrow tier
    int32_t route;                                          // diagonal tier: 0 no routing, 1 route_read decides, 2 route every unproved read
    const unsigned long long *n_dev;                        // launch over a list: *n_dev reads (entries of pair_order)
    int32_t vstride, hstride;
    const uint32_t *stage_src;        // = refs[0].prof2 (global source of the staged tile)
    int32_t stage_bytes;              // bytes of refs[0].prof2 staged into shared memory by TMA at kernel start (0: none)
    const uint8_t *lut;               // [256] ASCII -> alphabet code, 255 = not in the alphabet (device memory, L1-resident)
    int32_t phase_sync;               // g > 0: sets of g consecutive warps of a CTA walk through the per-group phases in step
                                      // (instruction-cache locality; a power of two dividing the CTA's warp count); 0: free-running warps
    const uint64_t *forced_ops;       // c2b_classify_aligned: op streams supplied by the caller, [read][32]
    const int32_t *forced_n;
};

// output slot of (read, reference): [read][ref] -- or [read][0] when every read carries its single reference (ref_id)
C2B_DEV int64_t oslot(const KParams &P, int64_t rd, int r) { return rd * P.out_refs + (P.ref_id ? 0 : r); }
// number of reads of this launch: a host constant, or (general kernel over the ALIGN kernel's left-over list) a device value
C2B_DEV int64_t nreads(const KParams &P) { return P.n_dev ? (int64_t)*P.n_dev : P.n_reads; }

// (A copy of the single reference's descriptor inside the kernel parameters was tried: no gain.)
C2B_DEV const RefDev &refdev(const KParams &P, int r) { return P.refs[r]; }

struct WarpSmem {
    uint8_t fw[2][MAXJ];       // read(s) as alphabet codes ([1]: second read of a pair)
    uint8_t rc[2][MAXJ];       // reverse complement
    uint8_t combo[MAXJ];       // pair path: codeA*nq + codeB of the strands being aligned
    uint8_t rowinfo[MAXI];     // per reference position: read code of its column, or 8 = deleted (pair: halves of 512)
    uint32_t rowins[MAXI + 4]; // rowins[r]: bases inserted between reference positions r-1 and r (pair: halves of 514)
};
constexpr int PK_ROWINFO_STRIDE = 512, PK_ROWINS_STRIDE = 514, PK_MAX_ALN = 512, PK_MAX_ALN2 = 1024;
// Ring-banded path: four pairs per warp, eight lanes each.  A group's lane r (0..7) plays the virtual lanes r, r+8, r+16, ...
// (virtual lane L = rows 8L+1..8L+8) one after the other, each for the RG_NS wavefront steps around its diagonal
// (step t -> slot t - 9L + RG_B); cells with column - row in [-(RG_B+1), RG_NS-RG_B-9] are always inside the band.
constexpr int RG_NS = 72, RG_B = 32, RG_MAXD = 8, RG_COMBO = 320;
constexpr int RG_MAX_REFS = 4, RG_OPS_STRIDE = 36;          // multi-reference ring path: references per read; u64 per (reference, pair): 32 op words + (n, err) of each half
constexpr int RG_DLO = RG_B + 1, RG_DHI = RG_NS - RG_B - 9;
struct QuadSmem {                                  // per warp; the op streams take the place of the base-pair codes once the DP is done
    union {
        uint8_t combo[4][RG_COMBO];
        struct { uint64_t ops[4][32]; int32_t n[4][2], err[4][2]; } wk;
    };
};
// Banded traceback slab of the packed path.  Lane l (rows 8l+1..8l+8) keeps only the PK_BAND_SLOTS wavefront steps around
// its own diagonal (step t -> slot t - 9l + PK_BAND_B): cells whose column is within about -29..+27 of their row.  The DP
// itself is unchanged (every cell is computed); if the traceback ever needs a cell outside the band, the pair is simply
// re-run with the full slab.  The banded slabs of the whole grid (16 KB per warp: ~35 MB for the 2112 resident warps of an H100) fit its 50 MB L2.
constexpr int PK_BAND_SLOTS = 64, PK_BAND_B = 28, PK_BAND_MAXD = 8;
// slot = t - slope*lane + off, kept iff 0 <= slot < ns.  Entry index: slot*32 + lane; ring slabs: (gb + (lane & 7))*TS + t,
// i.e. a lane's steps are consecutive (a diagonal run of the walk touches two or three 32-byte sectors).
struct SlabMode { int slope, off, ns, ring, gb; };

// ops: the lane's 32 columns of the op stream (lane L of the group: columns 32L..32L+31 from the right); ops2 (pair walks only):
// columns 512 + 32L.. of alignments longer than 512 columns (r02g: the ALIGN kernel takes pairs with I + J up to PK_MAX_ALN2)
struct Walked { uint64_t ops; int n; int err; uint64_t ops2; };

// ------------------------------------------------------------------------------------------------ DP
// Traceback word of (lane l, column j): bits [16+2k, 17+2k] = origin of M[i][j] (0 M, 1 J, 2 I) and bits
// [2k, 2k+1] = (bit 1: I[i][j] extends an I gap, bit 0: J[i][j] extends a J gap) for row i = 8l+k+1.
template <int KSTAR>
C2B_DEV void dp_block(const KParams &P, const RefDev &R, const uint8_t *codes, const int J, const int rb, const int NEG4,
                      uint32_t *__restrict__ tb, const int32_t *bnd_in, int32_t *bnd_out, int &cM, int &cX, int &cY)
{
    const int lane = wp::lane();
    const int nrb = R.nrb, lstar = R.lstar, Ipad = R.Ipad, gi0_4 = R.gi0_4;
    const bool lastblk = (rb == nrb - 1);
    const int nl = lastblk ? lstar + 1 : 32;
    const int rowbase = rb * 256;
    const int r0 = rowbase + 8 * lane;
    const bool islast = lastblk && lane == lstar;
    const int ge4 = 4 * P.ge, d4 = 4 * (P.go - P.ge);

    int M[8], X[8], Y[8], cIe[8], g4[8];
    {
        const int4 *pc = reinterpret_cast<const int4 *>(R.cIe + r0);
        const int4 *pg = reinterpret_cast<const int4 *>(R.g4 + r0);
        int4 a = wp::ldg4(pc), b = wp::ldg4(pc + 1), c = wp::ldg4(pg), d = wp::ldg4(pg + 1);
        cIe[0] = a.x; cIe[1] = a.y; cIe[2] = a.z; cIe[3] = a.w; cIe[4] = b.x; cIe[5] = b.y; cIe[6] = b.z; cIe[7] = b.w;
        g4[0] = c.x; g4[1] = c.y; g4[2] = c.z; g4[3] = c.w; g4[4] = d.x; g4[5] = d.y; g4[6] = d.z; g4[7] = d.w;
    }
#pragma unroll
    for (int k = 0; k < 8; k++) {          // column 0 (Align.pyx:153-176)
        M[k] = NEG4; X[k] = NEG4 | 2; Y[k] = (ge4 * (r0 + k + 1) + gi0_4) | 1;
    }
    int pM, pX, pY;                         // row above my first row, previous column (the diagonal of k=0)
    if (rb == 0) { pM = 0; pX = NEG4 | 2; pY = NEG4 | 1; }
    else { pM = NEG4; pX = NEG4 | 2; pY = (ge4 * rowbase + gi0_4) | 1; }

    const int nsteps = J + nl - 1;
    const int32_t *__restrict__ prof0 = R.prof + r0;
    uint32_t *__restrict__ tbw = tb + ((int64_t)rb * P.TS) * 32 + lane;
    const bool lane_on = lane < nl;
    int topX = gi0_4 | 2;                   // row 0: X[0][j] = 4*(ge*j + gi0) | 2, advanced by one column per step

    for (int t = 1; t <= nsteps; t++) {
        int uM = wp::shfl_up(M[7], 1), uX = wp::shfl_up(X[7], 1), uY = wp::shfl_up(Y[7], 1);
        const int j = t - lane;
        if (lane == 0) {
            if (rb == 0) { topX += ge4; uM = NEG4; uX = topX; uY = NEG4 | 1; }
            else if (j <= J) { uM = wp::ldcgi(bnd_in + 3 * j); uX = wp::ldcgi(bnd_in + 3 * j + 1); uY = wp::ldcgi(bnd_in + 3 * j + 2); }
        }
        if (lane_on && j >= 1 && j <= J) {
            const int q = codes[j - 1];
            const int4 *pp = reinterpret_cast<const int4 *>(prof0 + q * Ipad);
            const int4 sa = wp::ldg4(pp), sb = wp::ldg4(pp + 1);
            const int s[8] = {sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w};
            const int dcol = (j == J) ? 0 : d4;             // free opening in the last column (Align.pyx:234-273)
            const int dsp = islast ? 0 : dcol;              // ... and in the last row (:277-317)
            int dM = pM, dX = pX, dY = pY;
            int upM = uM, upY = uY;
            uint32_t wT = 0, wIJ = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const int dik = (k == KSTAR) ? dsp : dcol;
                const int z = wp::max3(dM, dY, dX);                      // diagonal, tie order I > J > M
                const int tag = z & 3;
                const int nm = (z - tag) + s[k];
                const int x = wp::addmax(M[k], dik, X[k]) + cIe[k];      // gap in reference ("I"), incentive of row i
                const int y = wp::addmax(upM, dik + g4[k], upY) + ge4;   // gap in read ("J"), incentive of row i-1 on open
                wT = wp::funnel_r(wT, (uint32_t)z, 2);                   // low two bits of z = origin of M
                wIJ = wp::funnel_r(wIJ, (uint32_t)(x | y), 2);   // low bits of x: 00/10 (I extends), of y: 00/01 (J extends)
                dM = M[k]; dX = X[k]; dY = Y[k];
                M[k] = nm; X[k] = x | 2; Y[k] = y | 1;
                upM = nm; upY = Y[k];
            }
            tbw[(int64_t)t * 32] = (wT & 0xffff0000u) | (wIJ >> 16);
            if (!lastblk && lane == 31) { bnd_out[3 * j] = M[7]; bnd_out[3 * j + 1] = X[7]; bnd_out[3 * j + 2] = Y[7]; }
        }
        pM = uM; pX = uX; pY = uY;
    }
    if (lastblk) {
        const int k = (KSTAR < 8) ? KSTAR : 0;
        cM = wp::shfl(M[k], lstar); cX = wp::shfl(X[k], lstar); cY = wp::shfl(Y[k], lstar);
    }
}

C2B_DEV void dp_dispatch(const KParams &P, const RefDev &R, const uint8_t *codes, int J, int rb, int NEG4,
                         uint32_t *tb, const int32_t *bi, int32_t *bo, int &cM, int &cX, int &cY)
{
    const int ks = (rb == R.nrb - 1) ? R.kstar : 8;
    switch (ks) {
    case 0: dp_block<0>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    case 1: dp_block<1>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    case 2: dp_block<2>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    case 3: dp_block<3>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    case 4: dp_block<4>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    case 5: dp_block<5>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    case 6: dp_block<6>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    case 7: dp_block<7>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    default: dp_block<8>(P, R, codes, J, rb, NEG4, tb, bi, bo, cM, cX, cY); break;
    }
}

// ------------------------------------------------------------------------------------------- traceback
// Batched traceback.  The walk of Align.pyx:338-421 moves along one direction per state (M: diagonal, J: up,
// I: left) and keeps that state while a per-cell bit says "continue" (M: origin tag is M; J/I: the gap extends).
// A group of G lanes therefore fetches the G next cells of the current direction in one gather, a ballot finds
// the first cell that breaks the run, and the whole run is consumed in one iteration (a read that matches its
// amplicon needs I/G iterations instead of I).  PAIR: lanes 0-15 walk read A and lanes 16-31 read B (G = 16,
// 64-bit slab entries); otherwise the 32 lanes walk one read (G = 32).  Output as before: the group's lane L holds
// ops 32L..32L+31 (2 bits each, counted from the right end of the alignment).
template <bool PAIR>
C2B_DEV Walked walk_batch(const KParams &P, const RefDev &R, const int J, const uint32_t *__restrict__ tb, int s, const SlabMode sm)
{
    const int lane = wp::lane();
    const int hl = PAIR ? (lane & 15) : lane, hb = PAIR ? (lane & 16) : 0;
    const int G = PAIR ? 16 : 32;
    const uint32_t gmask = PAIR ? 0xffffu : 0xffffffffu;
    const int TS = P.TS;
    const uint2 *__restrict__ tb2 = reinterpret_cast<const uint2 *>(tb);
    int i = R.I, j = J, n = 0, err = 0;
    uint32_t acc = 0, lo = ~0u, hi = ~0u, lo2 = ~0u, hi2 = ~0u;
    // 16 ops fill one 32-bit half-word; half-word ix belongs to word ix >> 1 = lane (word & (G-1)), second word when word >= G
    auto put = [&](int ix, uint32_t a) {
        const int word = ix >> 1;
        if (hl == (word & (G - 1))) {
            if (PAIR && word >= G) { if (ix & 1) hi2 = a; else lo2 = a; }
            else { if (ix & 1) hi = a; else lo = a; }
        }
    };
    // append `cnt` (<= 32) copies of op to the stream; acc holds the (n & 15) newest ops in its top bits
    auto push = [&](int op, int cnt) {
        const uint32_t pat = (uint32_t)op * 0x55555555u;
        while (cnt > 0) {
            const int room = 16 - (n & 15);
            const int c = cnt < room ? cnt : room;
            acc = (uint32_t)((((uint64_t)pat << 32) | acc) >> (2 * c));
            n += c; cnt -= c;
            if ((n & 15) == 0) put((n >> 4) - 1, acc);
        }
    };
    for (;;) {
        const bool active = i > 0 && j > 0;
        if (!wp::ballot(active)) break;
        const int di = (s != OP_I), dj = (s != OP_J);
        const int ci = i - hl * di, cj = j - hl * dj;
        const bool valid = active && ci >= 1 && cj >= 1;
        uint32_t v = 0;
        bool inband = valid;
        if (valid) {
            const int r = ci - 1, key = r >> 3, rb = key >> 5, l = key & 31;
            const int slot = cj + l - sm.slope * l + sm.off;
            inband = (unsigned)slot < (unsigned)sm.ns;
            if (inband) {
                const int64_t idx = sm.ring ? (int64_t)(sm.gb + (l & 7)) * TS + cj + l : ((int64_t)rb * TS + slot) * 32 + l;
                if (PAIR) {
                    const uint2 w2 = wp::ldcg2(tb2 + idx);
                    const uint32_t w = hb ? ((w2.x & 0xffff0000u) | (w2.y >> 16)) : ((w2.x << 16) | (w2.y & 0xffffu));
                    v = w >> (2 * (7 - (r & 7)));
                } else v = wp::ldcg(tb + idx) >> (2 * (r & 7));
            }
        }
        const int tag = (int)((v >> 16) & 3u);
        const bool cont = valid && (s == OP_M ? tag == OP_M : (v & (uint32_t)s) != 0u);
        const uint32_t bc = (wp::ballot(cont) >> hb) & gmask, bv = (wp::ballot(valid) >> hb) & gmask;
        const uint32_t bo = (wp::ballot(valid && !inband) >> hb) & gmask;      // cells the banded slab did not keep
        int nvalid = wp::popc(bv);                          // valid lanes are a prefix of the group
        if (bo) { const int fo = wp::ffs(bo) - 1; if (fo < nvalid) nvalid = fo; }
        const bool miss = active && nvalid == 0;            // the banded slab did not keep the next cell: caller re-runs with the full slab
        int f = wp::ffs(~bc) - 1;                           // leading run of "continue" (ffs(0) = 0 -> -1 when all 32 set)
        if (f < 0 || f > nvalid) f = nvalid;
        const bool brk = f < nvalid;
        const int run = brk ? f + 1 : nvalid;
        const int tagf = wp::shfl(tag, hb + (f < G ? f : G - 1));
        if (miss) { err |= 4; i = 0; j = 0; }
        else if (active) {
            const int news = brk ? (s == OP_M ? tagf : OP_M) : s;
            push(s, run);
            i -= run * di; j -= run * dj;
            err |= (news == 3);
            s = news;
            if (s == OP_M && sm.ring) {                     // ring slab: the next but one window (two lanes' worth of consecutive entries)
                const int pi = i - 2 * G - hl, pj = j - 2 * G - hl;
                if (pi >= 1 && pj >= 1 && (hl & 3) == 0) {
                    const int l = (pi - 1) >> 3;
                    wp::prefetch_l2(tb2 + (int64_t)(sm.gb + (l & 7)) * TS + pj + l);
                }
            } else if (s == OP_M && sm.slope == 0) {        // full slab: pull the window two iterations down the diagonal towards L2
                const int pi = i - 2 * G - hl, pj = j - 2 * G - hl;
                if (pi >= 1 && pj >= 1) {
                    const int r = pi - 1, key = r >> 3, rb = key >> 5, l = key & 31;
                    const int64_t idx = ((int64_t)rb * TS + pj + l) * 32 + l;
                    wp::prefetch_l2(PAIR ? (const void *)(tb2 + idx) : (const void *)(tb + idx));
                }
            }
        }
    }
    if (j > 0 && s != OP_I) err = 1;                        // row 0 / column 0 can only be left along their own border
    if (i > 0 && s != OP_J) err = 1;
    if (j > 0) { while (j > 0) { const int c = j < 32 ? j : 32; push(OP_I, c); j -= c; } }
    if (i > 0) { while (i > 0) { const int c = i < 32 ? i : 32; push(OP_J, c); i -= c; } }
    if (n & 15) {
        const int used = 2 * (n & 15);
        put(n >> 4, (acc >> (32 - used)) | (~0u << used));
    }
    if (n > (PAIR ? PK_MAX_ALN2 : 1024)) err |= 8;          // more columns than the stream holds (excluded by the callers' length limits)
    Walked out; out.ops = (uint64_t)lo | ((uint64_t)hi << 32); out.ops2 = (uint64_t)lo2 | ((uint64_t)hi2 << 32); out.n = n; out.err = err;
    return out;
}

// Full alignment of one strand against one reference: DP over row blocks, then the walk.
C2B_DEV Walked align_strand(const KParams &P, const RefDev &R, const uint8_t *codes, int J,
                            uint32_t *tb, int32_t *bnd)
{
    const int NEG4 = 4 * (int)((int64_t)P.go * J * R.I);        // sentinel of Align.pyx:150, scaled
    int cM = 0, cX = 0, cY = 0;
    const int bstride = 3 * (P.TS);
    const int nrb = R.nrb;
    for (int rb = 0; rb < nrb; rb++) {
        dp_dispatch(P, R, codes, J, rb, NEG4, tb, bnd + ((rb + 1) & 1) * bstride, bnd + (rb & 1) * bstride, cM, cX, cY);
        wp::sync();
    }
    const int s = wp::max3(cM, cY, cX) & 3;                     // start state, Align.pyx:349-358
    const SlabMode full = {0, 0, P.TS, 0, 0};
    return walk_batch<false>(P, R, J, tb, s, full);
}

// --------------------------------------------------------------------------------------------- columns
// mode bits: 1 = write strings, 2 = scatter per-reference-position info into shared memory.
// HALF = false: the warp's 32 lanes hold one read's op stream (lane L: columns 32L..32L+31 from the right).
// HALF = true : lanes 0-15 hold read A's stream, lanes 16-31 read B's (pair path); every argument is per lane.
struct ColOut { int n_match; int irregular; };

template <bool HALF>
C2B_DEVNOINL ColOut columns(const KParams &P, const RefDev &R, uint8_t *rowinfo, uint32_t *rowins, const uint8_t *codes, int J,
                            uint64_t ops, int n, int mode, uint8_t *out_read, uint8_t *out_ref)
{
    const int lane = wp::lane();
    const int li = HALF ? (lane & 15) : lane;            // lane index within the group that holds this read
    const uint64_t lo = 0x5555555555555555ull;
    const int ci = 32 - wp::popcll((ops >> 1) & lo);     // ops consuming a reference base (M, J)
    const int cj = 32 - wp::popcll(ops & lo);            // ops consuming a read base (M, I)
    int pk = (ci << 16) | cj;
#pragma unroll
    for (int d = 1; d < (HALF ? 16 : 32); d <<= 1) { int v = wp::shfl_up(pk, d); if (li >= d) pk += v; }
    pk -= (ci << 16) | cj;                               // exclusive
    int i = R.I - (pk >> 16), j = J - (pk & 0xffff);
    int match = 0, irr = 0;
    const int n0 = 32 * li;
    if (n0 < n) {
        // Right-aligned slots: column n (from the right) lives at byte W-1-n, so the lane's 32 columns are one
        // contiguous 32-byte sector, written as 8 aligned words (4 columns each).  The loop is deliberately not
        // unrolled 32x: this code runs once per read and must not evict the DP loop from the instruction cache.
        uint32_t *pr = (mode & 1) ? reinterpret_cast<uint32_t *>(out_read + P.W - n0 - 4) : nullptr;
        uint32_t *pf = (mode & 1) ? reinterpret_cast<uint32_t *>(out_ref + P.W - n0 - 4) : nullptr;
        uint64_t rest = ops;
#pragma unroll 1
        for (int w = 0; w < 8; w++) {
            uint32_t wr = 0, wf = 0;
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const int op = (int)rest & 3;
                rest >>= 2;
                if (op != OP_NONE) {
                    const int code = (op != OP_J) ? codes[j - 1] : 0;
                    const uint32_t rd = (op == OP_J) ? (uint32_t)'-' : (uint32_t)P.alpha[code];
                    const uint32_t rf = (op == OP_I) ? (uint32_t)'-' : (uint32_t)R.asc[i - 1];
                    if (op == OP_M && rd == rf) match++;
                    const int nn = n0 + 4 * w + e;
                    if ((nn == 0 || nn == n - 1) && (op != OP_M || rd != rf)) irr = 1;   // CRISPRessoCORE.py:729-733
                    wr |= rd << (8 * (3 - e)); wf |= rf << (8 * (3 - e));
                    if (mode & 2) {
                        if (op == OP_M) rowinfo[i - 1] = (uint8_t)code;
                        else if (op == OP_J) rowinfo[i - 1] = 8;
                        else if (i > 0 && i < R.I) wp::adds(&rowins[i], 1u);
                    }
                    i -= (op != OP_I); j -= (op != OP_J);
                }
            }
            if ((mode & 1) && n0 + 4 * w < n) { pr[-w] = wr; pf[-w] = wf; }
        }
    }
#pragma unroll
    for (int d = (HALF ? 8 : 16); d >= 1; d >>= 1) { match += wp::shfl_xor(match, d); irr |= wp::shfl_xor(irr, d); }
    ColOut o; o.n_match = match; o.irregular = irr;
    return o;
}

// exact round(100*m/n, 3)*1000 with Python's round-half-even (ties are exactly representable, DESIGN.md)
C2B_DEV int score_milli(int m, int n)
{
    // m <= n <= C2B_MAX_ALN_LEN = 1024: 100000*m < 2^27, so 32-bit unsigned arithmetic is exact (and the division is a
    // fraction of the 64-bit one's code)
    const uint32_t num = 100000u * (uint32_t)m, d = (uint32_t)n;
    uint32_t q = num / d; const uint32_t r = num - q * d;
    if (2u * r > d || (2u * r == d && (q & 1u))) q++;
    return (int)q;
}

// ------------------------------------------------------------------------------------------------ rows
struct RowOut {
    int ins_n, del_n, sub_n, n_ins_all, n_ins_win, n_del_all, n_del_win, n_del_pos, n_sub_all, nent;
};
// --coding_seq (CRISPRessoCORE.py:4104-4131): bases inserted by window insertions with a flank in an exon, any such
// insertion, deleted exon positions of window deletions, any window substitution in an exon, any window edit on a
// splicing position
struct CodOut { int ins_len, ins_any, del_cnt, sub_any, splice; };

// mode bits of rows_run
constexpr int RM_SCAL = 1;   // scalars + edit list (COREResources.pyx:108-163)
constexpr int RM_VEC = 2;    // per-position count vectors, weight w (CRISPRessoCORE.py:4016-4081)
constexpr int RM_LEN = 4;    // insertion/deletion length vectors (:4104-4115), only for reads that carry a modification
constexpr int RM_REF1 = 8;   // HDR re-projection (:4255-4272): the scattered alignment is the one to reference 0, the
                             // vectors updated are the ref1_* block of the reference the read was assigned to (Vt)

C2B_DEVNOINL void rows_run(const KParams &P, const RefDev &R, const uint8_t *rowinfo, const uint32_t *rowins, RowOut &o,
                           c2b_edit *ed, long long w, int mode, unsigned long long *Vt = nullptr)
{
    const int lane = wp::lane();
    const uint32_t lt = (1u << lane) - 1u;
    const bool ign_s = P.flags & C2B_F_IGNORE_SUBSTITUTIONS, ign_i = P.flags & C2B_F_IGNORE_INSERTIONS,
               ign_d = P.flags & C2B_F_IGNORE_DELETIONS;
    const bool scal = mode & RM_SCAL, vec = mode & RM_VEC, lenv = mode & RM_LEN, ref1 = mode & RM_REF1;
    unsigned long long *V = ref1 ? Vt : R.vec;
    const int vs = P.vstride;
    int open_a = -1; uint32_t prevD = 0;
    const int I = R.I;
    const int nchunks = (I + 32) >> 5;                    // covers position I itself (end of a trailing deletion)

    // --use_legacy_insertion_quantification (COREResources.pyx:190-315): an insertion is in the window when EITHER flank is
    // (:284); a deletion run is reported from reference position 0 when it starts in alignment column 0 or 1 (:252-254: a <= 1,
    // an insertion column never precedes a deletion column) and up to the LAST reference index, not one past it, when it reaches
    // the last column (:255-257: b == I); its size stays the column count.
    const bool legacy = (P.flags & C2B_F_LEGACY_INS) != 0;
    auto run = [&](int a0, int b0) {                       // one deletion run [a0,b0)  (COREResources.pyx:143-160)
        const int size = b0 - a0;
        const int a = (legacy && a0 <= 1) ? 0 : a0, b = (legacy && b0 == I) ? I - 1 : b0;
        const int npos = b > a ? b - a : 0;
        const bool hit = npos > 0 && (int)R.cum[b] - (int)R.cum[a] > 0;
        if (scal) {
            o.n_del_all++; o.n_del_pos += npos;
            if (hit) { o.n_del_win++; o.del_n += size; }
            if (lane == 0 && o.nent < P.edit_cap && ed) {
                c2b_edit e; e.a = (uint16_t)a; e.b = (uint16_t)b; e.type = 3; e.in_window = hit; e.pad = 0;
                e.base = legacy ? (uint8_t)(size - (b - a) + 2) : 0;            // legacy: size = b - a + base - 2
                ed[o.nent] = e;
            }
            o.nent++;
        }
        if (legacy && (vec || ref1))                       // all_deletion_positions = the reported range, not the deleted columns
            for (int p = a + lane; p < b; p += 32) wp::addg(V + (int64_t)(ref1 ? C2B_V_R1_ALL_DEL : C2B_V_ALL_DEL) * vs + p, w);
        if (hit && ((vec && !ign_d) || lenv)) {
            for (int p = a + lane; p < b; p += 32) {
                if (vec && !ign_d) wp::addg(V + (int64_t)C2B_V_DEL * vs + p, w);
                if (lenv) wp::addg(V + (int64_t)C2B_V_DEL_LEN * vs + p, w * size);
            }
        }
    };

    for (int c = 0; c < nchunks; c++) {
        const int p = 32 * c + lane;
        const bool valid = p < I;
        const int info = valid ? rowinfo[p] : 0;
        const bool isdel = valid && info == 8;
        const int rcode = info & 7;
        const uint32_t refc = valid ? R.asc[p] : 0u, readc = P.alpha[rcode];
        const bool differs = valid && !isdel && readc != refc;
        const uint32_t insr = (valid && p + 1 <= I - 1) ? rowins[p + 1] : 0u;   // insertion right of p
        const uint32_t insl = (valid && p >= 1 && p <= I - 1) ? rowins[p] : 0u; // insertion left of p
        // a chunk in which the read equals the reference and no deletion is open has nothing to record
        if (!wp::ballot(isdel || differs || insr > 0 || insl > 0) && !prevD) continue;
        const bool issub = differs && readc != 'N';                         // COREResources.pyx:111
        const bool inc_p = valid && (R.incl[p] & 1u);
        const bool win_r = insr > 0 && (legacy ? (inc_p || (R.incl[p + 1] & 1u)) : (inc_p && (R.incl[p + 1] & 1u)));   // both flanks in window (:120); legacy: either (:284)
        const bool win_l = insl > 0 && (legacy ? (inc_p || (R.incl[p - 1] & 1u)) : (inc_p && (R.incl[p - 1] & 1u)));
        const uint32_t D = wp::ballot(isdel);
        if (scal) {
            const uint32_t Bs = wp::ballot(issub), Bsw = wp::ballot(issub && inc_p);
            const uint32_t Bi = wp::ballot(insr > 0), Biw = wp::ballot(win_r);
            o.n_sub_all += wp::popc(Bs); o.sub_n += wp::popc(Bsw);
            o.n_ins_all += wp::popc(Bi); o.n_ins_win += wp::popc(Biw);
            if (Biw) {
                int v = win_r ? (int)insr : 0;
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) v += wp::shfl_xor(v, d);
                o.ins_n += v;
            }
            if (Bs) {
                const int idx = o.nent + wp::popc(Bs & lt);
                if (issub && idx < P.edit_cap && ed) {
                    c2b_edit e; e.a = (uint16_t)p; e.b = 0; e.type = 1; e.in_window = inc_p; e.base = (uint8_t)readc; e.pad = 0;
                    ed[idx] = e;
                }
                o.nent += wp::popc(Bs);
            }
            if (Bi) {
                const int idx = o.nent + wp::popc(Bi & lt);
                if (insr > 0 && idx < P.edit_cap && ed) {
                    c2b_edit e; e.a = (uint16_t)p; e.b = (uint16_t)insr; e.type = 2; e.in_window = win_r; e.base = 0; e.pad = 0;
                    ed[idx] = e;
                }
                o.nent += wp::popc(Bi);
            }
        }
        if (vec) {
            if (insr > 0) wp::addg(V + (int64_t)C2B_V_ALL_INS_LEFT * vs + p, w);
            if (insr > 0 || insl > 0) wp::addg(V + (int64_t)C2B_V_ALL_INS * vs + p, w);   // a shared flank counts once
            if (!ign_i && (win_r || win_l)) wp::addg(V + (int64_t)C2B_V_INS * vs + p, w);
            if (isdel && !legacy) wp::addg(V + (int64_t)C2B_V_ALL_DEL * vs + p, w);
            if (issub) {
                wp::addg(V + (int64_t)C2B_V_ALL_SUB * vs + p, w);
                if (!ign_s) {
                    wp::addg(V + (int64_t)(C2B_V_SUBBASE0 + rcode) * vs + p, w);
                    if (inc_p) wp::addg(V + (int64_t)C2B_V_SUB * vs + p, w);
                }
            }
            if (isdel || differs) {                       // all_base_count_vectors as deviation from "read == ref"
                const int rc = R.rcode[p];
                wp::addg(V + (int64_t)(C2B_V_BASEDEV0 + (isdel ? P.nq : rcode)) * vs + p, w);
                if (rc != 255) wp::addg(V + (int64_t)(C2B_V_BASEDEV0 + rc) * vs + p, -w);
            }
        }
        if (ref1) {
            if (insr > 0) wp::addg(V + (int64_t)C2B_V_R1_ALL_INS_LEFT * vs + p, w);
            if (insr > 0 || insl > 0) wp::addg(V + (int64_t)C2B_V_R1_ALL_INS * vs + p, w);
            if (isdel && !legacy) wp::addg(V + (int64_t)C2B_V_R1_ALL_DEL * vs + p, w);
            if (issub) wp::addg(V + (int64_t)C2B_V_R1_ALL_SUB * vs + p, w);
            if (isdel || differs) {
                const int rc = R.rcode[p];
                wp::addg(V + (int64_t)(C2B_V_R1_BASEDEV0 + (isdel ? P.nq : rcode)) * vs + p, w);
                if (rc != 255) wp::addg(V + (int64_t)(C2B_V_R1_BASEDEV0 + rc) * vs + p, -w);
            }
        }
        if (lenv && (win_r || win_l))
            wp::addg(V + (int64_t)C2B_V_INS_LEN * vs + p, w * (long long)((win_r ? insr : 0u) + (win_l ? insl : 0u)));
        // deletion runs: ends inside this chunk
        const uint32_t Dsh = (D << 1) | prevD;
        const uint32_t Sm = D & ~Dsh;
        uint32_t E = ~D & Dsh;
        uint32_t Erem = E;
        while (Erem) {
            const int eb = wp::ffs(Erem) - 1;
            Erem &= Erem - 1;
            const uint32_t below = Sm & ((1u << eb) - 1u);
            const int a = below ? 32 * c + (31 - wp::clz(below)) : open_a;
            run(a, 32 * c + eb);
        }
        if (D >> 31) {
            const int hs = Sm ? 31 - wp::clz(Sm) : -1, he = E ? 31 - wp::clz(E) : -1;
            if (hs > he) open_a = 32 * c + hs;
        }
        prevD = D >> 31;
    }
    if (prevD) run(open_a, I);
}

// --coding_seq part of the quantification loop (CRISPRessoCORE.py:4104-4171), kept out of rows_run so that the hot
// per-read code does not grow: a second scan of the same row-space view, run only for reads of a reference with a
// coding sequence that enter that block.  add_noncoding = false: fill `c`; true: add the window edit positions of a
// read that touches no exon to the *_noncoding vectors (:4166-4170).
C2B_DEVNOINL void rows_coding(const KParams &P, const RefDev &R, const uint8_t *rowinfo, const uint32_t *rowins, CodOut &c,
                              long long w, bool add_noncoding)
{
    const int lane = wp::lane();
    unsigned long long *V = R.vec;
    const int vs = P.vstride, I = R.I;
    const int nchunks = (I + 32) >> 5;
    int open_a = -1; uint32_t prevD = 0;
    auto run = [&](int a, int b) {
        if ((int)R.cum[b] - (int)R.cum[a] <= 0) return;        // deletion_positions holds runs that touch the window
        if (!add_noncoding) {
            c.del_cnt += (int)R.cumx[b] - (int)R.cumx[a];
            if ((int)R.cums[b] - (int)R.cums[a] > 0) c.splice = 1;
        } else for (int p = a + lane; p < b; p += 32) wp::addg(V + (int64_t)C2B_V_DEL_NONCODING * vs + p, w);
    };
    for (int ch = 0; ch < nchunks; ch++) {
        const int p = 32 * ch + lane;
        const bool valid = p < I;
        const int info = valid ? rowinfo[p] : 0;
        const bool isdel = valid && info == 8;
        const uint32_t refc = valid ? R.asc[p] : 0u, readc = P.alpha[info & 7];
        const bool issub = valid && !isdel && readc != refc && readc != 'N';
        const uint32_t insr = (valid && p + 1 <= I - 1) ? rowins[p + 1] : 0u;
        const uint32_t insl = (valid && p >= 1 && p <= I - 1) ? rowins[p] : 0u;
        const uint32_t mk = valid ? R.incl[p] : 0u, mk1 = insr > 0 ? R.incl[p + 1] : 0u;
        const bool inc_p = mk & 1u;
        const bool win_r = insr > 0 && inc_p && (mk1 & 1u);
        const bool win_l = insl > 0 && inc_p && (R.incl[p - 1] & 1u);
        if (!add_noncoding) {
            const bool xi = win_r && ((mk | mk1) & 2u);        // window insertion with a flank in an exon
            if (wp::ballot(xi)) {
                int v = xi ? (int)insr : 0;
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) v += wp::shfl_xor(v, d);
                c.ins_len += v; c.ins_any = 1;
            }
            if (wp::ballot(issub && inc_p && (mk & 2u))) c.sub_any = 1;
            if (wp::ballot((issub && inc_p && (mk & 4u)) || (win_r && ((mk | mk1) & 4u)))) c.splice = 1;
        } else {
            if (win_r || win_l) wp::addg(V + (int64_t)C2B_V_INS_NONCODING * vs + p, w);
            if (issub && inc_p) wp::addg(V + (int64_t)C2B_V_SUB_NONCODING * vs + p, w);
        }
        const uint32_t D = wp::ballot(isdel);
        const uint32_t Dsh = (D << 1) | prevD;
        const uint32_t Sm = D & ~Dsh;
        uint32_t E = ~D & Dsh;
        uint32_t Erem = E;
        while (Erem) {
            const int eb = wp::ffs(Erem) - 1;
            Erem &= Erem - 1;
            const uint32_t below = Sm & ((1u << eb) - 1u);
            run(below ? 32 * ch + (31 - wp::clz(below)) : open_a, 32 * ch + eb);
        }
        if (D >> 31) {
            const int hs = Sm ? 31 - wp::clz(Sm) : -1, he = E ? 31 - wp::clz(E) : -1;
            if (hs > he) open_a = 32 * ch + hs;
        }
        prevD = D >> 31;
    }
    if (prevD) run(open_a, I);
}

// Frameshift / splicing decision of CRISPRessoCORE.py:4117-4171 for one counted read of a coding reference.
C2B_DEVNOINL void coding_update(const KParams &P, const RefDev &R, const uint8_t *rowinfo, const uint32_t *rowins,
                                bool has_window_edits, long long w)
{
    CodOut c; c.ins_len = c.ins_any = c.del_cnt = c.sub_any = c.splice = 0;
    rows_coding(P, R, rowinfo, rowins, c, w, false);
    const int lm = c.ins_len - c.del_cnt;                     // sum(length_modified_positions_exons)
    const bool exmod = c.ins_any || c.del_cnt > 0 || c.sub_any;
    int slot, row, key = 0;
    if (R.tem != 0 || (exmod && (c.ins_any || c.del_cnt > 0))) {
        key = lm + R.tem;
        const bool inframe = key % 3 == 0;
        slot = inframe ? C2B_S_MOD_NON_FRAMESHIFT : C2B_S_MOD_FRAMESHIFT;
        row = inframe ? C2B_H_INFRAME : C2B_H_FRAMESHIFT;
    } else if (exmod) { slot = C2B_S_MOD_NON_FRAMESHIFT; row = C2B_H_INFRAME; }
    else {
        slot = C2B_S_NON_MOD_NON_FRAMESHIFT; row = C2B_H_INFRAME;
        if (has_window_edits) rows_coding(P, R, rowinfo, rowins, c, w, true);
    }
    if (wp::lane() == 0) {
        wp::addg(R.scal + slot, w);
        wp::addg(R.hist + (int64_t)row * P.hstride + R.hist_zero + key, w);
        if (c.splice) wp::addg(R.scal + C2B_S_SPLICING_MODIFIED, w);
    }
}

// What only edited reads (or reads of a reference whose exons changed length) add to the count block once they are
// counted: the size Counters (CRISPRessoCORE.py:4020-4043; the commonest bucket is implied, see c2b200.h), the
// insertion/deletion/substitution class counters (:4022-4072) and the --coding_seq decision.  Inline: measured faster than
// an out-of-line call, although two thirds of the reads never get here.
C2B_DEV void edited_update(const KParams &P, const RefDev &R, const uint8_t *rowinfo, const uint32_t *rowins,
                           const RowOut &o, long long w)
{
    const bool ign_s = P.flags & C2B_F_IGNORE_SUBSTITUTIONS, ign_i = P.flags & C2B_F_IGNORE_INSERTIONS,
               ign_d = P.flags & C2B_F_IGNORE_DELETIONS;
    if (R.coding) coding_update(P, R, rowinfo, rowins, o.n_ins_win > 0 || o.n_del_win > 0 || o.sub_n > 0, w);
    if (wp::lane() != 0) return;
    const bool has_d = !ign_d && o.del_n > 0, has_i = !ign_i && o.ins_n > 0, has_s = !ign_s && o.sub_n > 0;
    unsigned long long *H = R.hist, *SC = R.scal;
    const int hs = P.hstride;
    if (has_i) wp::addg(H + (int64_t)C2B_H_INS_N * hs + o.ins_n, w);
    if (has_d) wp::addg(H + (int64_t)C2B_H_DEL_N * hs + o.del_n, w);
    if (has_s) wp::addg(H + (int64_t)C2B_H_SUB_N * hs + o.sub_n, w);
    const int eff = R.I + (has_i ? o.ins_n : 0) - (has_d ? o.del_n : 0);
    if (eff != R.I) wp::addg(H + (int64_t)C2B_H_EFF_LEN * hs + eff, w);
    if (has_i) wp::addg(SC + C2B_S_INS, w);
    if (has_d) wp::addg(SC + C2B_S_DEL, w);
    if (has_s) wp::addg(SC + C2B_S_SUB, w);
    const int combo = (has_i ? 4 : 0) | (has_d ? 2 : 0) | (has_s ? 1 : 0);
    const int slot[8] = {-1, C2B_S_ONLY_SUB, C2B_S_ONLY_DEL, C2B_S_DEL_SUB, C2B_S_ONLY_INS, C2B_S_INS_SUB,
                         C2B_S_INS_DEL, C2B_S_INS_DEL_SUB};
    if (slot[combo] >= 0) wp::addg(SC + slot[combo], w);
}

// ------------------------------------------------------------------------------------------ per read
C2B_DEV int strand_mode(const KParams &P, const RefDev &R, const uint8_t *fw, int J)
{
    // seed test of CRISPRessoCORE.py:656-687: 0 forward only, 1 reverse-complement only, 2 both
    if (P.flags & C2B_F_NO_STRAND_SEARCH) return 0;
    const int lane = wp::lane();
    const int L = R.seed_len, ns = R.nseeds;
    uint32_t hit = 0;                                        // bit s: fw seed s seen ; bit 8+s: rc seed s seen
    if (ns > 0 && L > 0) {
        // each lane owns 8 consecutive start positions per 256-position block: roll the packed k-mer along them into
        // registers first, then compare every seed (loaded once) against the 8 k-mers
        const uint64_t top = 3 * (uint64_t)(L - 1);
        for (int base = 8 * lane; base + L <= J; base += 256) {
            uint64_t km[8];
            uint64_t cur = 0;
            for (int c = 0; c < L; c++) cur |= (uint64_t)fw[base + c] << (3 * c);
#pragma unroll
            for (int e = 0; e < 8; e++) {
                km[e] = (base + e + L <= J) ? cur : ~0ull;                 // ~0 never equals a seed
                if (e < 7 && base + e + L < J) cur = (cur >> 3) | ((uint64_t)fw[base + e + L] << top);
            }
#pragma unroll 1
            for (int s = 0; s < ns; s++) {
                const uint64_t f = R.fw_seed[s], r = R.rc_seed[s];
                bool hf = false, hr = false;
#pragma unroll
                for (int e = 0; e < 8; e++) { hf |= (km[e] == f); hr |= (km[e] == r); }
                if (hf && f != ~0ull) hit |= 1u << s;
                if (hr && r != ~0ull) hit |= 1u << (8 + s);
            }
        }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) hit |= (uint32_t)wp::shfl_xor((int)hit, d);
    const int nf = wp::popc(hit & 0xffu), nr = wp::popc(hit >> 8);
    if (nf > P.seed_min && nr == 0) return 0;
    if (nf == 0 && nr > P.seed_min) return 1;
    return 2;
}

// read -> alphabet codes (forward and reverse complement); returns true if a symbol is outside the alphabet
C2B_DEV bool load_codes(const KParams &P, int64_t off, int J, uint8_t *fw, uint8_t *rc)
{
    const int lane = wp::lane();
    bool bad = false;
    for (int base = 0; base < J; base += 256) {             // 8 symbols per lane per round: all loads first, then use
        uint8_t ch[8];
#pragma unroll
        for (int e = 0; e < 8; e++) { const int p = base + lane + 32 * e; ch[e] = p < J ? P.reads[off + p] : (uint8_t)P.alpha[0]; }
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const int p = base + lane + 32 * e;
            int code = P.lut[ch[e]];
            if (code == 255) { bad = true; code = 0; }
            if (p < J) { fw[p] = (uint8_t)code; rc[J - 1 - p] = P.comp[code]; }
        }
    }
    return wp::ballot(bad) != 0;
}

C2B_DEV void init_aln(c2b_aln_rec &a, uint32_t st)
{
    a.n_match = 0; a.aln_len = 0; a.score_milli = -1000; a.strand = 0; a.status = (uint8_t)st; a.n_edits = 0;
    a.insertion_n = a.deletion_n = a.substitution_n = 0; a.n_ins_all = a.n_ins_win = 0; a.n_del_all = a.n_del_win = 0;
    a.n_del_pos_all = 0; a.n_sub_all = 0; a.irregular_ends = 0; a.modified = 0;
}

// best-reference bookkeeping of CRISPRessoCORE.py:697-707
C2B_DEV void note_score(c2b_read_rec &rec, const RefDev &R, int r, int sc)
{
    if (sc > rec.best_score_milli && (double)sc / 1000.0 > R.min_aln) {
        rec.best_score_milli = sc; rec.winner_mask = 1u << (r & 31); rec.n_winners = 1;
    } else if (sc == rec.best_score_milli) {
        rec.winner_mask |= 1u << (r & 31); rec.n_winners++;
    }
}

// c2b_aln_rec written by another lane of this warp: read it through L2 (the writer's line may sit stale in L1)
C2B_DEV c2b_aln_rec load_aln(const c2b_aln_rec *p)
{
    union { c2b_aln_rec a; uint64_t q[4]; } u;
    const uint64_t *s = reinterpret_cast<const uint64_t *>(p);
    u.q[0] = wp::ldcg64(s); u.q[1] = wp::ldcg64(s + 1); u.q[2] = wp::ldcg64(s + 2); u.q[3] = wp::ldcg64(s + 3);
    return u.a;
}

C2B_DEV void sc_add(unsigned long long *SC, int slot, long long v) { wp::addg(SC + slot, v); }

// Several references were tried: reload the op stream of the read's alignment to reference r (kept in opsbuf; lane offset
// hoff >= 0: the stream lives in 16 lanes starting at hoff) and scatter it into the row-space view again.  -> irregular_ends
C2B_DEVNOINL int rescatter(const KParams &P, const RefDev &R, int64_t rd, int r, const uint64_t *opsbuf, int hoff,
                           uint8_t *rowinfo, uint32_t *rowins, const uint8_t *fw, const uint8_t *rc, int J)
{
    const int lane = wp::lane();
    wp::sync();
    uint64_t ops;
    if (hoff < 0) ops = wp::ldcg64(opsbuf + r * 32 + lane);
    else ops = lane < 16 ? wp::ldcg64(opsbuf + r * 32 + hoff + lane) : ~0ull;
    const c2b_aln_rec prev = load_aln(P.alns + oslot(P, rd, r));
    const int n = wp::shfl((int)prev.aln_len, 0), strand = wp::shfl((int)prev.strand, 0);
    const int irr = wp::shfl((int)prev.irregular_ends, 0);
    for (int p = lane; p <= R.I; p += 32) rowins[p] = 0;
    wp::sync();
    columns<false>(P, R, rowinfo, rowins, strand ? rc : fw, J, ops, n, 2, nullptr, nullptr);
    return irr;
}

// Classification + counts of one read once its alignments are known (all lanes hold the same `rec`).
//   single reference tried: the caller already scattered the chosen alignment into rowinfo/rowins;
//   several references    : op streams are reloaded from opsbuf (lane offset hoff; hoff >= 0: the stream lives in
//                           16 lanes starting at hoff) and re-scattered per winner.
// ONE: one candidate reference per read (a single amplicon, or Pooled ref_id) -- a compile-time fact of the launch, so that
// the lean kernel carries none of the several-references code (loops over winners, re-scatter, HDR re-projection).
template <bool ONE>
C2B_DEV void finish_read(const KParams &P, int64_t rd, c2b_read_rec rec, int J, const uint8_t *fw, const uint8_t *rc,
                         uint8_t *rowinfo, uint32_t *rowins, int r_begin, int r_end, const uint64_t *opsbuf, int hoff,
                         int keep_irr, const c2b_aln_rec &a_single)
{
    const int lane = wp::lane();
    const bool multi = !ONE && (r_end - r_begin) > 1;
    if (ONE) r_end = r_begin + 1;
    if (rec.best_score_milli <= 0 && !P.forced_ops) { rec.winner_mask = 0; rec.n_winners = 0; }
    else {
        const bool expand = P.flags & C2B_F_EXPAND_AMBIGUOUS, first = P.flags & C2B_F_ASSIGN_FIRST;
        const bool ambiguous = !ONE && rec.n_winners > 1 && !first && !expand;     // CRISPRessoCORE.py:780-785
        rec.ambiguous = ambiguous;
        const long long cnt = P.count ? P.count[rd] : 1;
        const long long w = P.qweight ? P.qweight[rd] : cnt;
        int nth = 0;
        for (int r = r_begin; r < r_end; r++) {
            if (!((rec.winner_mask >> (r & 31)) & 1u)) continue;
            const RefDev &R = refdev(P, r);
            rec.best_ref = (int16_t)r;                          // best_match_name = last winner (:768)
            int irr = keep_irr;
            if (multi) irr = rescatter(P, R, rd, r, opsbuf, hoff, rowinfo, rowins, fw, rc, J);
            wp::sync();
            RowOut o; o.ins_n = o.del_n = o.sub_n = 0; o.n_ins_all = o.n_ins_win = o.n_del_all = o.n_del_win = 0;
            o.n_del_pos = o.n_sub_all = 0; o.nent = 0;
            c2b_edit *ed = P.edits ? P.edits + oslot(P, rd, r) * (int64_t)P.edit_cap : nullptr;
            const bool ign_s = P.flags & C2B_F_IGNORE_SUBSTITUTIONS, ign_i = P.flags & C2B_F_IGNORE_INSERTIONS,
                       ign_d = P.flags & C2B_F_IGNORE_DELETIONS;
            // contribution to the count block (CRISPRessoCORE.py:3989-4072); known before the scan unless
            // --discard_indel_reads is on, in which case the scalars decide and the vectors need a second scan
            const bool counted = !ambiguous && (!first || nth == 0) && w > 0;
            const bool two_scans = (P.flags & C2B_F_DISCARD_INDEL_READS) != 0;
            rows_run(P, R, rowinfo, rowins, o, ed, w, RM_SCAL | ((counted && !two_scans) ? RM_VEC : 0));
            const bool has_d = !ign_d && o.del_n > 0, has_i = !ign_i && o.ins_n > 0, has_s = !ign_s && o.sub_n > 0;
            const bool modified = has_d || has_i || has_s;     // CRISPRessoCORE.py:746-753 (same truth table)
            uint32_t astatus = 0;
            if (P.edits && o.nent > P.edit_cap) astatus |= C2B_ST_EDIT_OVERFLOW;     // list truncated; counts are complete
            unsigned long long *SC = R.scal;
            if (counted) {
                const bool discard = two_scans && (o.del_n > 0 || o.ins_n > 0);
                if (discard) { if (lane == 0) sc_add(SC, C2B_S_DISCARDED, w); }
                else {
                    // the block of CRISPRessoCORE.py:4085-4171 is entered by modified reads, and by every read of a reference
                    // whose exons changed length (tot_exon_len_mod != 0)
                    const bool entered = modified || R.tem != 0;
                    const bool lenv = entered && (o.n_ins_win > 0 || o.n_del_win > 0);
                    if (two_scans || lenv) rows_run(P, R, rowinfo, rowins, o, nullptr, w, (two_scans ? RM_VEC : 0) | (lenv ? RM_LEN : 0));
                    if (entered) edited_update(P, R, rowinfo, rowins, o, w);     // everything only edited reads add (out of line)
                    if (lane == 0) {
                        sc_add(SC, C2B_S_TOTAL, w);
                        sc_add(SC, modified ? C2B_S_MODIFIED : C2B_S_UNMODIFIED, w);
                    }
                }
            } else if (ambiguous && nth == 0 && w > 0 && lane == 0) sc_add(SC, C2B_S_AMBIGUOUS_W, w);
            // class_counts (:3984-3986) as a deviation from counts_modified / counts_unmodified: a discarded read still has
            // its class; a counted winner of an --expand_ambiguous_alignments read with several winners has a joined label
            // (derived on the host) instead
            if (counted && lane == 0 && (two_scans || expand)) {
                const bool discarded = two_scans && (o.del_n > 0 || o.ins_n > 0), joined = !ONE && expand && !first && rec.n_winners > 1;   // assign-first is tested first (:780-785)
                if (discarded != joined) sc_add(SC, modified ? C2B_S_CLASS_MODIFIED : C2B_S_CLASS_UNMODIFIED, discarded ? w : -w);
            }
            if (lane == 0) {
                c2b_aln_rec a = multi ? load_aln(P.alns + oslot(P, rd, r)) : a_single;   // single reference: still in registers
                a.insertion_n = (uint16_t)o.ins_n; a.deletion_n = (uint16_t)o.del_n; a.substitution_n = (uint16_t)o.sub_n;
                a.n_ins_all = (uint16_t)o.n_ins_all; a.n_ins_win = (uint16_t)o.n_ins_win;
                a.n_del_all = (uint16_t)o.n_del_all; a.n_del_win = (uint16_t)o.n_del_win;
                a.n_del_pos_all = (uint16_t)o.n_del_pos; a.n_sub_all = (uint16_t)o.n_sub_all;
                a.n_edits = (uint16_t)o.nent; a.modified = modified; a.status |= (uint8_t)astatus;
                a.irregular_ends = (uint8_t)irr;
                P.alns[oslot(P, rd, r)] = a;
            }
            rec.status |= astatus;
            nth++;
            // aln_stats of the serial process_fastq branch use best_match_name only (:1971-1979): the LAST winner
            const bool is_last = (rec.winner_mask >> (r & 31)) >> 1 == 0;
            if (is_last && lane == 0) {
                const long long total_mods = o.n_ins_all + o.n_del_pos + o.n_sub_all;
                const long long in_win = o.sub_n + o.del_n + o.ins_n;
                sc_add(SC, C2B_S_N_GLOBAL_SUBS, cnt * o.n_sub_all);
                sc_add(SC, C2B_S_N_SUBS_OUTSIDE_WINDOW, cnt * (o.n_sub_all - o.sub_n));
                sc_add(SC, C2B_S_N_MODS_IN_WINDOW, cnt * in_win);
                sc_add(SC, C2B_S_N_MODS_OUTSIDE_WINDOW, cnt * (total_mods - in_win));
                if (irr) sc_add(SC, C2B_S_N_READS_IRREGULAR_ENDS, cnt);
                sc_add(SC, C2B_S_N_ALIGNED_UNIQUE, 1);
                sc_add(SC, C2B_S_N_ALIGNED_COUNT, cnt);
            }
            wp::sync();
        }
        // HDR / prime editing: reads assigned to another reference are also classified on their alignment to reference 0
        if (!ONE && (P.flags & C2B_F_HDR_REF1) && multi && r_begin == 0 && !ambiguous && w > 0) {
            const uint32_t eff = first ? (rec.winner_mask & (0u - rec.winner_mask)) : rec.winner_mask;   // aln_ref_names
            if (eff != 1u) {                                    // not "aligned to reference 0 only" (:4234)
                const RefDev &R0 = P.refs[0];
                rescatter(P, R0, rd, 0, opsbuf, hoff, rowinfo, rowins, fw, rc, J);
                wp::sync();
                RowOut dummy; dummy.ins_n = dummy.del_n = dummy.sub_n = 0; dummy.n_ins_all = dummy.n_ins_win = 0;
                dummy.n_del_all = dummy.n_del_win = dummy.n_del_pos = dummy.n_sub_all = 0; dummy.nent = 0;
                for (int r = 1; r < r_end; r++) {
                    if (!((eff >> (r & 31)) & 1u)) continue;
                    rows_run(P, R0, rowinfo, rowins, dummy, nullptr, w, RM_REF1, P.refs[r].vec);
                    if (lane == 0) wp::addg(P.refs[r].scal + C2B_S_REF1_W, w);
                }
                wp::sync();
            }
        }
    }
    if (lane == 0) P.recs[rd] = rec;
}

// One read per warp, 32-bit scores: the general path (any length within the build limits, any parameters).
template <bool ONE>
C2B_DEV void process_read(const KParams &P, WarpSmem &S, int64_t rd, int warp_slot)
{
    const int lane = wp::lane();
    const int64_t off = P.offsets[rd];
    const int J = (int)(P.offsets[rd + 1] - off);
    uint32_t *tb = P.tb + (int64_t)warp_slot * P.tb_words_per_warp;
    int32_t *bnd = P.bnd + (int64_t)warp_slot * P.bnd_words_per_warp;
    uint64_t *opsbuf = P.opsbuf + (int64_t)warp_slot * P.ops_refs * 32;

    c2b_read_rec rec; rec.winner_mask = 0; rec.best_score_milli = -1000; rec.best_ref = -1; rec.n_winners = 0;
    rec.ambiguous = 0; rec.status = 0;
    uint32_t st = 0;
    if (J < 1 || J > MAXJ || J + 32 > P.TS) st |= C2B_ST_TOO_LONG;
    else if (load_codes(P, off, J, S.fw[0], S.rc[0])) st |= C2B_ST_BAD_CHAR;
    wp::sync();

    const int r_begin = P.ref_id ? P.ref_id[rd] : 0;
    const int r_end = (ONE || P.ref_id) ? r_begin + 1 : P.n_refs;
    const bool multi = !ONE && (r_end - r_begin) > 1;
    int keep_irr = 0;
    c2b_aln_rec a; init_aln(a, st);

    for (int r = r_begin; r < r_end; r++) {
        const RefDev &R = refdev(P, r);
        init_aln(a, st);
        if (!st && (R.I + J > C2B_MAX_ALN_LEN)) a.status |= C2B_ST_TOO_LONG;
        if (!a.status) {
            const int mode = P.forced_ops ? 0 : strand_mode(P, R, S.fw[0], J);
            Walked wf; wf.ops = ~0ull; wf.n = 0; wf.err = 0;
            Walked wr = wf;
            int sf = -1000000, sr = -1000000;
            for (int pass = 0; pass < 2; pass++) {              // one call site: forward, then reverse complement
                if (pass == (mode == 1 ? 0 : mode == 0 ? 1 : 2)) continue;
                const uint8_t *codes = pass ? S.rc[0] : S.fw[0];
                Walked wk;
                if (P.forced_ops) { wk.ops = P.forced_ops[rd * 32 + lane]; wk.n = P.forced_n[rd]; wk.err = 0; }
                else wk = align_strand(P, R, codes, J, tb, bnd);
                int sc = -1000000;
                if (wk.err) a.status |= C2B_ST_UNDEFINED;
                else if (mode == 2) sc = score_milli(columns<false>(P, R, S.rowinfo, S.rowins, codes, J, wk.ops, wk.n, 0, nullptr, nullptr).n_match, wk.n);
                if (pass) { wr = wk; sr = sc; } else { wf = wk; sf = sc; }
            }
            if (!a.status) {
                const bool use_rc = (mode == 1) || (mode == 2 && sr > sf);      // strict '>' of CRISPRessoCORE.py:682
                const Walked &wk = use_rc ? wr : wf;
                const uint8_t *codes = use_rc ? S.rc[0] : S.fw[0];
                uint8_t *o_read = P.strings ? P.strings + (oslot(P, rd, r) * 2) * (int64_t)P.W : nullptr;
                uint8_t *o_ref = o_read ? o_read + P.W : nullptr;
                int cmode = (o_read ? 1 : 0);
                if (!multi) {                                   // single reference: scatter now, classify below
                    for (int p = lane; p <= R.I; p += 32) S.rowins[p] = 0;
                    wp::sync();
                    cmode |= 2;
                }
                const ColOut co = columns<false>(P, R, S.rowinfo, S.rowins, codes, J, wk.ops, wk.n, cmode, o_read, o_ref);
                a.n_match = (uint16_t)co.n_match; a.aln_len = (uint16_t)wk.n; a.strand = use_rc;
                a.score_milli = score_milli(co.n_match, wk.n);
                a.irregular_ends = (uint8_t)co.irregular;
                if (multi) opsbuf[r * 32 + lane] = wk.ops;
                if (P.gops && !P.forced_ops) {
                    if (lane < P.NW) P.gops[oslot(P, rd, r) * P.NW + lane] = wk.ops;
                    if (lane == 0) P.gmeta[oslot(P, rd, r)] = (uint32_t)wk.n | ((uint32_t)use_rc << 16) | (2u << 24);
                }
                if (lane == 0) wp::maxg(&P.wb->launch.widest, (unsigned long long)wk.n);   // widest alignment of the launch
                keep_irr = co.irregular;
                note_score(rec, R, r, a.score_milli);
            }
        }
        rec.status |= a.status;
        if (lane == 0) P.alns[oslot(P, rd, r)] = a;
    }
    wp::sync();
    finish_read<ONE>(P, rd, rec, J, S.fw[0], S.rc[0], S.rowinfo, S.rowins, r_begin, r_end, opsbuf, -1, keep_irr, a);
}

// ------------------------------------------------------------------------------------ paired path (16-bit halves)
// Two reads of equal length share a warp: every 32-bit register holds read A's value in its low half and read
// B's in its high half, so each VIMNMX3.S16x2 / VIADDMNMX.S16x2 advances two DP cells.  Scores are biased by
// beta*(i+j) (beta = -gap_extend; equal for all values compared at one cell, so every decision is unchanged) plus a
// constant offset, which makes every stored value and every added constant non-negative: plain 32-bit adds then
// cannot carry between the halves.  Validity (ranges, parameter signs) is decided per reference on the host
// (RefDev::pk_maxJ); anything else takes the 32-bit path above.
constexpr uint32_t PK_SENT = 0x01000100u, PK_T2 = 0x00020002u, PK_T1 = 0x00010001u, PK_TM = 0x00030003u;

template <int KSTAR, bool STAGED>
C2B_DEV void dp_block2(const KParams &P, const RefDev &R, const uint32_t *prof, const uint8_t *combo, const int J, const int rb,
                       uint2 *__restrict__ tb2, const SlabMode sm, const int32_t *bnd_in, int32_t *bnd_out, uint32_t &cM, uint32_t &cX, uint32_t &cY)
{
    const int lane = wp::lane();
    const int nrb = R.nrb, lstar = R.lstar, Ipad = R.Ipad;
    const bool lastblk = (rb == nrb - 1);
    const int nl = lastblk ? lstar + 1 : 32;
    const int r0 = rb * 256 + 8 * lane;
    const bool islast = lastblk && lane == lstar;
    const uint32_t d4p = (uint32_t)((4 * (P.go - P.ge)) & 0xffff) * 0x00010001u;
    const uint32_t XB = R.pk_XB, YB = R.pk_YB;

    uint32_t M[8], X[8], Y[8], cIe[8], g4[8];
    {
        const uint4 *pc = reinterpret_cast<const uint4 *>(R.cIe2 + r0);
        const uint4 *pg = reinterpret_cast<const uint4 *>(R.g42 + r0);
        uint4 a = wp::ldg4u(pc), b = wp::ldg4u(pc + 1), c = wp::ldg4u(pg), d = wp::ldg4u(pg + 1);
        cIe[0] = a.x; cIe[1] = a.y; cIe[2] = a.z; cIe[3] = a.w; cIe[4] = b.x; cIe[5] = b.y; cIe[6] = b.z; cIe[7] = b.w;
        g4[0] = c.x; g4[1] = c.y; g4[2] = c.z; g4[3] = c.w; g4[4] = d.x; g4[5] = d.y; g4[6] = d.z; g4[7] = d.w;
    }
#pragma unroll
    for (int k = 0; k < 8; k++) { M[k] = PK_SENT; X[k] = PK_SENT | PK_T2; Y[k] = YB; }      // column 0
    uint32_t pM, pX, pY;
    if (rb == 0) { pM = R.pk_M00; pX = PK_SENT | PK_T2; pY = PK_SENT | PK_T1; }
    else { pM = PK_SENT; pX = PK_SENT | PK_T2; pY = YB; }

    const int nsteps = J + nl - 1;
    const uint32_t *__restrict__ prof0 = prof + rb * 256 + lane * 4;     // shared (TMA-staged) or global copy, same layout
    int slot = 1 - sm.slope * lane + sm.off;                             // slab slot of step t = 1 for this lane
    uint2 *__restrict__ tbp = tb2 + ((int64_t)rb * P.TS + slot) * 32 + lane;   // advanced by one slot (32 entries) per step
    const bool lane_on = lane < nl;

    for (int t = 1; t <= nsteps; t++) {
        uint32_t uM = wp::shflu_up(M[7], 1), uX = wp::shflu_up(X[7], 1), uY = wp::shflu_up(Y[7], 1);
        const int j = t - lane;
        if (lane == 0) {
            if (rb == 0) { uM = PK_SENT; uX = XB; uY = PK_SENT | PK_T1; }
            else if (j <= J) { uM = (uint32_t)wp::ldcgi(bnd_in + 3 * j); uX = (uint32_t)wp::ldcgi(bnd_in + 3 * j + 1); uY = (uint32_t)wp::ldcgi(bnd_in + 3 * j + 2); }
        }
        if (lane_on && j >= 1 && j <= J) {
            const uint4 *pp = reinterpret_cast<const uint4 *>(prof0 + combo[j - 1] * Ipad);
            const uint4 sa = pp[0], sb = pp[32];            // conflict-free 16-byte accesses (lanes contiguous per half)
            const uint32_t s[8] = {sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w};
            const uint32_t dcol = (j == J) ? 0u : d4p;      // free opening in the last column (both reads end together)
            const uint32_t dsp = islast ? 0u : dcol;
            uint32_t dM = pM, dX = pX, dY = pY, upM = uM, upY = uY, wT = 0, wIJ = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const uint32_t dik = (k == KSTAR) ? dsp : dcol;
                const uint32_t z = wp::max3_2(dM, dY, dX);
                const uint32_t t2 = z & PK_TM;
                const uint32_t nm = z - t2 + s[k];                                   // halves stay in [0, 32767]: no carry
                const uint32_t x = wp::addmax_2(M[k], dik, X[k]) + cIe[k];
                const uint32_t y = wp::addmax_2(upM + g4[k], dik, upY);              // biased gap_extend is 0
                wT = wT * 4u + t2;
                wIJ = wIJ * 4u + ((x | y) & PK_TM);     // x's low bits are 00/10 (I extends), y's 00/01 (J extends)
                dM = M[k]; dX = X[k]; dY = Y[k];
                M[k] = nm; X[k] = x | PK_T2; Y[k] = y | PK_T1;
                upM = nm; upY = Y[k];
            }
            if ((unsigned)slot < (unsigned)sm.ns) *tbp = make_uint2(wT, wIJ);
            if (!lastblk && lane == 31) { bnd_out[3 * j] = (int)M[7]; bnd_out[3 * j + 1] = (int)X[7]; bnd_out[3 * j + 2] = (int)Y[7]; }
        }
        tbp += 32; slot++;
        pM = uM; pX = uX; pY = uY;
    }
    if (lastblk) {
        const int k = (KSTAR < 8) ? KSTAR : 0;
        cM = wp::shflu(M[k], lstar); cX = wp::shflu(X[k], lstar); cY = wp::shflu(Y[k], lstar);
    }
}

template <bool STAGED>
C2B_DEV void dp_dispatch2(const KParams &P, const RefDev &R, const uint32_t *prof, const uint8_t *combo, int J, int rb, uint2 *tb2,
                          const SlabMode sm, const int32_t *bi, int32_t *bo, uint32_t &cM, uint32_t &cX, uint32_t &cY)
{
    const int ks = (rb == R.nrb - 1) ? R.kstar : 8;
    switch (ks) {
    case 0: dp_block2<0, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    case 1: dp_block2<1, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    case 2: dp_block2<2, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    case 3: dp_block2<3, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    case 4: dp_block2<4, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    case 5: dp_block2<5, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    case 6: dp_block2<6, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    case 7: dp_block2<7, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    default: dp_block2<8, STAGED>(P, R, prof, combo, J, rb, tb2, sm, bi, bo, cM, cX, cY); break;
    }
}

C2B_DEV Walked align_pair(const KParams &P, const RefDev &R, const uint32_t *prof, bool staged, const uint8_t *combo, int J,
                          uint2 *tb_full, uint2 *tb_band, int32_t *bnd)
{
    const int bstride = 3 * (P.TS);
    const int nrb = R.nrb;
    const int d = J - R.I;
    bool band = tb_band != nullptr && nrb == 1 && d >= -PK_BAND_MAXD && d <= PK_BAND_MAXD;
    for (;;) {
        const SlabMode sm = band ? SlabMode{9, PK_BAND_B, PK_BAND_SLOTS, 0, 0} : SlabMode{0, 0, P.TS, 0, 0};
        uint2 *tb2 = band ? tb_band : tb_full;
        uint32_t cM = 0, cX = 0, cY = 0;
        for (int rb = 0; rb < nrb; rb++) {
            if (staged) dp_dispatch2<true>(P, R, prof, combo, J, rb, tb2, sm, bnd + ((rb + 1) & 1) * bstride, bnd + (rb & 1) * bstride, cM, cX, cY);
            else dp_dispatch2<false>(P, R, prof, combo, J, rb, tb2, sm, bnd + ((rb + 1) & 1) * bstride, bnd + (rb & 1) * bstride, cM, cX, cY);
            wp::sync();
        }
        const uint32_t s2 = wp::max3_2(cM, cY, cX) & PK_TM;         // start state per half
        const int s = (wp::lane() & 16) ? (int)(s2 >> 16) : (int)(s2 & 3u);
        const Walked wk = walk_batch<true>(P, R, J, reinterpret_cast<const uint32_t *>(tb2), s, sm);
        if (!band || !wp::ballot((wk.err & 4) != 0)) return wk;
        band = false;                                               // a traceback left the band: once more with the full slab
        if (wp::lane() == 0) wp::addg(&P.wb->band_reruns, 1);
    }
}


// ------------------------------------------------------------------------------------ ring-banded path (four pairs per warp)
// Same packed arithmetic as dp_block2, but only the cells of a diagonal band are computed.  The warp is split into four
// rings of eight lanes, one pair of reads each.  Ring lane r plays virtual lanes r, r+8, r+16, ... (virtual lane L owns
// rows 8L+1..8L+8 and, at step t, column t-L) for RG_NS consecutive steps each; lane edges travel around the ring by
// shuffle, so the lower row block starts while the upper one is still running and no lane idles.  Cells outside the
// band read as the sentinel (never above the true value), hence every banded value is <= the full-matrix value and equal
// to it along any path that stays inside the band: if the banded score beats ring_bound() -- an upper bound on the score
// of every alignment that leaves the band -- the full-matrix traceback lies inside the band and the banded traceback
// reproduces it cell for cell (ties included).  Otherwise the pair takes align_pair() over the full matrix.
// Slab: entry (t, physical lane), one coalesced 256-byte row per step.
// RL = lanes per ring: 8 (four pairs per warp, band RG_NS = 72 slots) or 4 (eight pairs per warp, band 36 slots: the narrow
// first tier of r02i -- twice the reads per pass for reads whose alignment stays within about [-17, +11] of the diagonal).
template <bool STAGED, int RL = 8>
C2B_DEVNOINL void dp_ring(const KParams &P, const RefDev &R, const uint32_t *prof, const uint8_t *combo, const int J, const int nsteps,
                          uint2 *__restrict__ tbq, uint32_t *fin)
{
    constexpr int NS = 9 * RL, B = 4 * RL;                               // slots per window, slots left of the diagonal
    const int lane = wp::lane(), r8 = lane & (RL - 1);
    const int src = (lane & ~(RL - 1)) | ((lane + RL - 1) & (RL - 1));   // ring predecessor
    const int lstar = R.lstar;
    const uint32_t combo_sa = wp::smem_addr(combo) - 1u;                 // combo[j-1] = [combo_sa + j]
    const uint32_t qstride = (uint32_t)R.Ipad * 4u;
    // loop invariants read through R (global memory: the compiler re-loads them every step next to the slab stores)
    const int Ipad = R.Ipad, Iref = R.I;
    const uint32_t XB0 = R.pk_XB;

    uint32_t M[8], X[8], Y[8], cIe[8], g40, dI[8];                       // g4[k] = 4*gi[row] = cIe[k-1]; g40: the row above the lane's first
    int L = r8, slot = 1 - 9 * r8 + B;                                // slot of step t = 1
    uint32_t prof_sa = 0; const uint32_t *prof0 = prof;
    auto enter = [&](int Lv) {                                           // constants and left-of-band state of virtual lane Lv
        const int row0 = 8 * (Lv <= lstar ? Lv : lstar);                 // past the last row block: inert, any valid rows
        const uint4 *pc = reinterpret_cast<const uint4 *>(R.cIe2 + row0);
        const uint4 a = wp::ldg4u(pc), b = wp::ldg4u(pc + 1);
        cIe[0] = a.x; cIe[1] = a.y; cIe[2] = a.z; cIe[3] = a.w; cIe[4] = b.x; cIe[5] = b.y; cIe[6] = b.z; cIe[7] = b.w;
        g40 = R.g42[row0];
        const uint32_t y0 = (8 * Lv - B <= 0) ? R.pk_YB : (PK_SENT | PK_T1);   // window starts at column 0: the border column
        const uint32_t d4p = (uint32_t)((4 * (P.go - P.ge)) & 0xffff) * 0x00010001u;
        const int klast = Iref - 8 * Lv - 1;                              // row I is this lane's row klast (if 0 <= klast < 8)
#pragma unroll
        for (int k = 0; k < 8; k++) {
            M[k] = PK_SENT; X[k] = PK_SENT | PK_T2; Y[k] = y0;
            dI[k] = (k == klast) ? 0u : d4p;                             // free opening in the last row
        }
        if (STAGED) prof_sa = wp::smem_addr(prof) + (uint32_t)Lv * 16u; else prof0 = prof + Lv * 4;
    };
    enter(L);
    uint32_t pM = R.pk_M00, pX = PK_SENT | PK_T2, pY = PK_SENT | PK_T1;  // diagonal of (1,1); other lanes: carried below
    uint2 *__restrict__ tbp = tbq + (int64_t)lane * P.TS;                // this lane's entries; step t -> entry t, written two at a time
    uint32_t hT = 0, hIJ = 0;                                            // an even step's entry, held until the odd step
    bool pend = false;

    for (int t = 1; t <= nsteps; t++) {
        uint32_t uM = wp::shflu(M[7], src), uX = wp::shflu(X[7], src), uY = wp::shflu(Y[7], src);
        if (L == 0) { uM = PK_SENT; uX = XB0; uY = PK_SENT | PK_T1; }     // row 0
        const int j = t - L;
        if (slot >= 0 && L <= lstar && j >= 1 && j <= J) {
            uint32_t s[8];
            if (STAGED) {
                const uint32_t a = prof_sa + wp::lds_u8(combo_sa + (uint32_t)j) * qstride;
                const uint4 sa = wp::lds_v4(a), sb = wp::lds_v4(a + 512u);
                s[0] = sa.x; s[1] = sa.y; s[2] = sa.z; s[3] = sa.w; s[4] = sb.x; s[5] = sb.y; s[6] = sb.z; s[7] = sb.w;
            } else {
                const uint4 *pp = reinterpret_cast<const uint4 *>(prof0 + combo[j - 1] * Ipad);
                const uint4 sa = wp::ldg4u(pp), sb = wp::ldg4u(pp + 32);
                s[0] = sa.x; s[1] = sa.y; s[2] = sa.z; s[3] = sa.w; s[4] = sb.x; s[5] = sb.y; s[6] = sb.z; s[7] = sb.w;
            }
            const uint32_t cm = (j == J) ? 0u : 0xffffffffu;             // free opening in the last column
            // the row above leaves the band NS-8 slots into the window (its diagonal neighbour one slot later)
            const bool lateU = slot >= NS - 8, lateP = slot > NS - 8;
            uint32_t dM = lateP ? PK_SENT : pM, dX = lateP ? (PK_SENT | PK_T2) : pX, dY = lateP ? (PK_SENT | PK_T1) : pY;
            uint32_t upM = lateU ? PK_SENT : uM, upY = lateU ? (PK_SENT | PK_T1) : uY, wT = 0, wIJ = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const uint32_t dik = dI[k] & cm;
                const uint32_t z = wp::max3_2(dM, dY, dX);
                const uint32_t t2 = z & PK_TM;
                const uint32_t nm = z - t2 + s[k];
                const uint32_t x = wp::addmax_2(M[k], dik, X[k]) + cIe[k];
                const uint32_t y = wp::addmax_2(upM + (k ? cIe[k ? k - 1 : 0] : g40), dik, upY);
                wT = wT * 4u + t2;
                wIJ = wIJ * 4u + ((x | y) & PK_TM);
                dM = M[k]; dX = X[k]; dY = Y[k];
                M[k] = nm; X[k] = x | PK_T2; Y[k] = y | PK_T1;
                upM = nm; upY = Y[k];
            }
            if (t & 1) *reinterpret_cast<uint4 *>(tbp + (t - 1)) = make_uint4(hT, hIJ, wT, wIJ);
            hT = wT; hIJ = wIJ; pend = !(t & 1);
            if (j == J && L == lstar) {                                  // cell (I, J): the three final values
                const int kstar = R.kstar;
#pragma unroll
                for (int k = 0; k < 8; k++) if (k == kstar) { fin[3 * lane] = M[k]; fin[3 * lane + 1] = X[k]; fin[3 * lane + 2] = Y[k]; }
            }
        }
        else if (pend) { tbp[t - 1] = make_uint2(hT, hIJ); pend = false; }     // the active stretch ended on an even step
        pM = uM; pX = uX; pY = uY;                                       // raw: a lane entering its next window needs the uncapped edge
        if (++slot == NS) { L += RL; slot = 0; enter(L); }
    }
    if (pend) tbp[nsteps] = make_uint2(hT, hIJ);
}

// Upper bound on the score of any alignment of a J-long read that visits a cell with column - row outside
// [-RG_DLO, RG_DHI].  Such a path holds at least nh >= RG_DHI+1 read-only columns (and nv = nh - (J-I) reference-only
// ones) or nv >= RG_DLO+1 reference-only columns (and nh = nv + (J-I)); a gap column scores at most gap_extend (+ the
// largest incentive for read-only columns; reference-only runs collect each row's incentive at most once, gsum in
// total), a diagonal column at most smax.  The host proves the bound decreasing in the free count (RefDev::rg_ok).
C2B_DEV int ring_bound(const KParams &P, const RefDev &R, int J, const int DLO = RG_DLO, const int DHI = RG_DHI)
{
    const int I = R.I, D = J - I, ge = P.ge, smax = R.rg_smax, gmax = R.rg_gmax;
    int U = -(1 << 28);
    {
        int nh = DHI + 1; if (nh < D) nh = D;
        const int nv = nh - D;
        if (nh <= J && nv <= I) { const int u = smax * (J - nh) + nh * (ge + gmax) + nv * ge + R.rg_gsum; if (u > U) U = u; }
    }
    {
        int nv = DLO + 1; if (nv < -D) nv = -D;
        const int nh = nv + D;
        if (nv <= I && nh <= J && nh >= 0) { const int u = smax * (I - nv) + nh * (ge + gmax) + nv * ge + R.rg_gsum; if (u > U) U = u; }
    }
    return U;
}

// A pair aligned by dp_ring: its walked op streams, lengths, strand modes.  ref_stride == 0: one reference, streams in shared
// memory (ops/n/err).  ref_stride > 0: several references tried, reference k's block (RG_OPS_STRIDE u64, global scratch,
// written by this warp) starts at ops + k * ref_stride; refmask bit k = the band held for reference k.
struct RingCtx { const uint64_t *ops; const int32_t *n, *err; int modes; int ref_stride; uint32_t refmask; };
// Barriers per work group when the warps of a phase set move in step: 3 in process_quad / process_quad_multi, and per pair one
// at entry, two per reference tried (before its alignment pass and before its columns) and two for the classify steps.
// The same count for every warp of a launch (it depends on the configuration only), so warps on other paths execute that
// many empty barriers.
C2B_DEV int group_phases(const KParams &P) { const int nr = P.ref_id ? 1 : P.n_refs; return 3 + 4 * (3 + 2 * nr); }

// Two reads (rdA, rdB) of equal length J through the packed path.  Per-lane variables belong to the lane's half.
template <bool ONE>
C2B_DEVNOINL void process_pair(const KParams &P, WarpSmem &S, const uint32_t *staged_prof, int64_t rdA, int64_t rdB, int warp_slot,
                          const RingCtx *ring, const bool phased)
{
    // phased: called once per pair of a work group by every warp of the CTA -- PAIR_PHASES CTA barriers keep the warps in the
    // same stretch of code (the per-read path is larger than the instruction cache; see DESIGN.md section 3)
    if (phased) wp::grp_sync(P.phase_sync);
    const int lane = wp::lane(), h = lane >> 4, hl = lane & 15;
    const int64_t myrd = h ? rdB : rdA;
    const int J = (int)(P.offsets[rdA + 1] - P.offsets[rdA]);
    uint2 *tb2 = reinterpret_cast<uint2 *>(P.tb + (int64_t)warp_slot * P.tb_words_per_warp);
    uint2 *tbb = P.tbb ? reinterpret_cast<uint2 *>(P.tbb + (int64_t)warp_slot * P.tbb_words_per_warp) : nullptr;
    int32_t *bnd = P.bnd + (int64_t)warp_slot * P.bnd_words_per_warp;
    uint64_t *opsbuf = P.opsbuf + (int64_t)warp_slot * P.ops_refs * 32;
    uint8_t *rowinfo = S.rowinfo + h * PK_ROWINFO_STRIDE;
    uint32_t *rowins = S.rowins + h * PK_ROWINS_STRIDE;

    c2b_read_rec rec; rec.winner_mask = 0; rec.best_score_milli = -1000; rec.best_ref = -1; rec.n_winners = 0;
    rec.ambiguous = 0; rec.status = 0;
    uint32_t badmask = 0;
#pragma unroll 1
    for (int x = 0; x < 2; x++)                            // one copy of the loader in the instruction stream
        if (load_codes(P, P.offsets[x ? rdB : rdA], J, S.fw[x], S.rc[x])) badmask |= 1u << x;
    const uint32_t st = ((badmask >> h) & 1u) ? C2B_ST_BAD_CHAR : 0u;
    wp::sync();

    const int r_begin = P.ref_id ? P.ref_id[rdA] : 0;
    const int r_end = (ONE || P.ref_id) ? r_begin + 1 : P.n_refs;
    const bool multi = !ONE && (r_end - r_begin) > 1;
    int keep_irr = 0;
    c2b_aln_rec a; init_aln(a, st);

    for (int r = r_begin; r < r_end; r++) {
        const RefDev &R = refdev(P, r);
        init_aln(a, st);
        int mAB = 0;
        if (ring) mAB = ring->modes;
        else {
#pragma unroll 1
            for (int x = 0; x < 2; x++) mAB |= strand_mode(P, R, S.fw[x], J) << (2 * x);
        }
        const int mA = mAB & 3, mB = mAB >> 2;
        const int mode = h ? mB : mA;
        const int npass = (mA == 2 || mB == 2) ? 2 : 1;
        uint64_t bops = ~0ull; int bn = 0, bstrand = 0, bscore = -1000000;
        for (int pass = 0; pass < npass; pass++) {
            // strand of each read in this pass: a one-strand read repeats its only strand in pass 1 (result unused)
            const int sA = (mA == 2) ? pass : (mA == 1), sB = (mB == 2) ? pass : (mB == 1);
            const uint8_t *cA = sA ? S.rc[0] : S.fw[0], *cB = sB ? S.rc[1] : S.fw[1];
            wp::sync();
            if (phased && pass == 0) wp::grp_sync(P.phase_sync);
            Walked wk; wk.err = 4;
            if (ring && (ONE || ring->ref_stride == 0)) { wk.ops = ring->ops[lane]; wk.n = ring->n[h]; wk.err = ring->err[h]; }   // aligned and walked by process_quad
            else if (!ONE && ring && ((ring->refmask >> (r - r_begin)) & 1u)) {
                const uint64_t *o = ring->ops + (int64_t)(r - r_begin) * ring->ref_stride;
                wk.ops = wp::ldcg64(o + lane);
                const uint64_t mt = wp::ldcg64(o + 32 + h);
                wk.n = (int)(uint32_t)mt; wk.err = (int)(mt >> 32);
            }
            if (wk.err & 4) {
                for (int p = lane; p < J; p += 32) S.combo[p] = (uint8_t)(cA[p] * P.nq + cB[p]);
                wp::sync();
                const bool staged = (r == 0 && staged_prof != nullptr);
                wk = align_pair(P, R, staged ? staged_prof : R.prof2, staged, S.combo, J, tb2, tbb, bnd);
            }
            const int mystrand = h ? sB : sA;
            if (wk.err) a.status |= C2B_ST_UNDEFINED;
            int sc = -1000000;
            if (wp::ballot(mode == 2)) {
                const ColOut c0 = columns<true>(P, R, rowinfo, rowins, mystrand ? S.rc[h] : S.fw[h], J, wk.ops, wk.n, 0, nullptr, nullptr);
                sc = score_milli(c0.n_match, wk.n);
            }
            // pass 1 of a both-strand read is its reverse complement: it replaces the forward result only if strictly better
            if (pass == 0 || (mode == 2 && sc > bscore)) { bops = wk.ops; bn = wk.n; bstrand = mystrand; bscore = sc; }
        }
        for (int p = lane; p < 2 * PK_ROWINS_STRIDE; p += 32) S.rowins[p] = 0;
        wp::sync();
        if (phased) wp::grp_sync(P.phase_sync);
        uint8_t *o_read = P.strings ? P.strings + (oslot(P, myrd, r) * 2) * (int64_t)P.W : nullptr;
        uint8_t *o_ref = o_read ? o_read + P.W : nullptr;
        int cmode = (o_read ? 1 : 0) | (multi ? 0 : 2);
        if (a.status) cmode = 0;
        const ColOut co = columns<true>(P, R, rowinfo, rowins, bstrand ? S.rc[h] : S.fw[h], J, bops, bn, cmode, o_read, o_ref);
        if (!a.status) {
            a.n_match = (uint16_t)co.n_match; a.aln_len = (uint16_t)bn; a.strand = (uint8_t)bstrand;
            a.score_milli = score_milli(co.n_match, bn);
            a.irregular_ends = (uint8_t)co.irregular;
            keep_irr = co.irregular;
            note_score(rec, R, r, a.score_milli);
            if (hl == 0) wp::maxg(&P.wb->launch.widest, (unsigned long long)bn);
        }
        if (multi) opsbuf[r * 32 + lane] = bops;
        if (P.gops && !a.status && (h == 0 || rdB != rdA)) {
            if (hl < P.NW) P.gops[oslot(P, myrd, r) * P.NW + hl] = bops;
            if (hl == 0) P.gmeta[oslot(P, myrd, r)] = (uint32_t)bn | ((uint32_t)bstrand << 16) | (2u << 24);
        }
        rec.status |= a.status;
        if (hl == 0 && (h == 0 || rdB != rdA)) P.alns[oslot(P, myrd, r)] = a;
    }
    wp::sync();
    // classification runs with the whole warp, one read at a time: broadcast that half's bookkeeping to every lane.
    // (The compiler unrolls this loop into two copies of finish_read; forcing one copy, or making finish_read and the
    // loaders out-of-line calls, shrank the kernel but made it slower.)
    for (int hh = 0; hh < 2; hh++) {
        if (phased) wp::grp_sync(P.phase_sync);
        if (hh == 1 && rdB == rdA) break;
        const int src = 16 * hh;
        c2b_read_rec rr;
        rr.winner_mask = wp::shflu(rec.winner_mask, src); rr.best_score_milli = wp::shfl(rec.best_score_milli, src);
        rr.best_ref = -1; rr.n_winners = (uint8_t)wp::shfl((int)rec.n_winners, src); rr.ambiguous = 0;
        rr.status = wp::shflu(rec.status, src);
        const int irr = wp::shfl(keep_irr, src);
        c2b_aln_rec ah; init_aln(ah, 0);                    // that half's record (used when a single reference was tried)
        const uint32_t w0 = wp::shflu((uint32_t)a.n_match | ((uint32_t)a.aln_len << 16), src);
        ah.n_match = (uint16_t)(w0 & 0xffffu); ah.aln_len = (uint16_t)(w0 >> 16);
        ah.score_milli = wp::shfl(a.score_milli, src);
        const uint32_t w1 = wp::shflu((uint32_t)a.strand | ((uint32_t)a.status << 8), src);
        ah.strand = (uint8_t)(w1 & 0xffu); ah.status = (uint8_t)(w1 >> 8);
        finish_read<ONE>(P, hh ? rdB : rdA, rr, J, S.fw[hh], S.rc[hh], S.rowinfo + hh * PK_ROWINFO_STRIDE,
                    S.rowins + hh * PK_ROWINS_STRIDE, r_begin, r_end, opsbuf, src, irr, ah);
        wp::sync();
    }
}

// Work item w = reads 2w and 2w+1.  Equal lengths inside every reference's proven 16-bit range -> packed pair;
// otherwise each read takes the 32-bit path.
template <bool ONE>
C2B_DEV void process_item(const KParams &P, WarpSmem &S, const uint32_t *staged_prof, int64_t w, int warp_slot)
{
    const bool haveB = 2 * w + 1 < nreads(P);
    const int64_t rdA = P.pair_order ? P.pair_order[2 * w] : 2 * w;
    const int64_t rdB = haveB ? (P.pair_order ? P.pair_order[2 * w + 1] : 2 * w + 1) : rdA;
    bool pair = !P.forced_ops && !(P.flags & C2B_F_NO_PAIRING);
    if (pair) {
        const int Ja = (int)(P.offsets[rdA + 1] - P.offsets[rdA]);
        const int Jb = haveB ? (int)(P.offsets[rdB + 1] - P.offsets[rdB]) : Ja;
        pair = (Ja == Jb) && Ja >= 1 && Ja + 32 <= P.TS;
        if (pair && P.ref_id && haveB && P.ref_id[rdA] != P.ref_id[rdB]) pair = false;
        if (pair) {
            const int r_begin = P.ref_id ? P.ref_id[rdA] : 0, r_end = P.ref_id ? r_begin + 1 : P.n_refs;
            for (int r = r_begin; r < r_end; r++) if (Ja > refdev(P, r).pk_maxJ || refdev(P, r).I + Ja > PK_MAX_ALN) pair = false;
        }
    }
    if (wp::lane() == 0) wp::addg(pair ? &P.wb->pair_items : &P.wb->single_items, 1);      // path statistics (c2b_path_counts)
    if (pair) process_pair<ONE>(P, S, staged_prof, rdA, rdB, warp_slot, nullptr, false);
    else {
        process_read<ONE>(P, S, rdA, warp_slot);
        if (haveB && rdB != rdA) { wp::sync(); process_read<ONE>(P, S, rdB, warp_slot); }   // (rdA, rdA): a single read on the left-over list
    }
}


// Four equal-length pairs against one reference: strands and base-pair codes per pair, one ring-banded DP for all
// four, then every pair continues through process_pair (walk + classification) -- with the ring's slab if its score
// proves the band sufficient, over the full matrix otherwise.
C2B_DEV void process_quad(const KParams &P, WarpSmem &S, QuadSmem &Q, const uint32_t *staged_prof, int64_t first, int warp_slot)
{
    const int lane = wp::lane(), g = lane >> 3;
    uint2 *tbq = reinterpret_cast<uint2 *>(P.tbq + (int64_t)warp_slot * P.TS * 64);
    if (P.phase_sync) wp::grp_sync(P.phase_sync);
    uint32_t okmask = 0, modes = 0;
    int Jg = 0, Jmax = 0;
    const int64_t rd0 = P.pair_order ? P.pair_order[2 * first] : 2 * first;
    const int r = P.ref_id ? P.ref_id[rd0] : 0;
    const RefDev &R = refdev(P, r);
#pragma unroll 1
    for (int q = 0; q < 4; q++) {
        const int64_t rdA = P.pair_order ? P.pair_order[2 * (first + q)] : 2 * (first + q);
        const int64_t rdB = P.pair_order ? P.pair_order[2 * (first + q) + 1] : 2 * (first + q) + 1;
        const int J = (int)(P.offsets[rdA + 1] - P.offsets[rdA]);
        bool bad = false;
#pragma unroll 1
        for (int x = 0; x < 2; x++) bad |= load_codes(P, P.offsets[x ? rdB : rdA], J, S.fw[x], S.rc[x]);
        wp::sync();
        int mAB = 0;
#pragma unroll 1
        for (int x = 0; x < 2; x++) mAB |= strand_mode(P, R, S.fw[x], J) << (2 * x);
        const int mA = mAB & 3, mB = mAB >> 2;
        if (!bad && mA != 2 && mB != 2) {                   // a read that needs both strands takes the full path
            const uint8_t *cA = mA ? S.rc[0] : S.fw[0], *cB = mB ? S.rc[1] : S.fw[1];
            for (int p = lane; p < J; p += 32) Q.combo[q][p] = (uint8_t)(cA[p] * P.nq + cB[p]);
            okmask |= 1u << q; modes |= (uint32_t)mAB << (4 * q);
            if (g == q) Jg = J;
            if (J > Jmax) Jmax = J;
        }
        wp::sync();
    }
    uint32_t passmask = 0, s2 = 0;
    if (P.phase_sync) wp::grp_sync(P.phase_sync);
    if (okmask) {
        const bool staged = (r == 0 && staged_prof != nullptr);
        uint32_t *fin = S.rowins;                            // 32 x 3 words: each ring's final lane leaves M, X, Y of cell (I, J)
        if (staged) dp_ring<true>(P, R, staged_prof, Q.combo[g], Jg, Jmax + R.lstar, tbq, fin);
        else dp_ring<false>(P, R, R.prof2, Q.combo[g], Jg, Jmax + R.lstar, tbq, fin);
        wp::sync();
        const int fl = 3 * ((lane & 24) | (R.lstar & 7));
        const uint32_t cM = Jg > 0 ? fin[fl] : PK_SENT, cX = Jg > 0 ? fin[fl + 1] : PK_SENT, cY = Jg > 0 ? fin[fl + 2] : PK_SENT;
        wp::sync();
        const uint32_t z = wp::max3_2(cM, cY, cX);
        s2 = z & PK_TM;
        // biased value = 4*(score + beta*(I+J) + 512) + tag: both reads must beat the out-of-band bound
        const int thr = ring_bound(P, R, Jg) + 512 - P.ge * (R.I + Jg);
        const bool pass = Jg > 0 && (int)((z & 0xffffu) >> 2) > thr && (int)(z >> 18) > thr;
        const uint32_t b = wp::ballot(pass);
        passmask = (b & 1u) | ((b >> 7) & 2u) | ((b >> 14) & 4u) | ((b >> 21) & 8u);
    }
    if (P.phase_sync) wp::grp_sync(P.phase_sync);
    // the four tracebacks while the slab is still warm in L2; the op streams replace the base-pair codes in shared memory
#pragma unroll 1
    for (int q = 0; q < 4; q++) {
        if (!((passmask >> q) & 1u)) continue;
        const uint32_t sq = wp::shflu(s2, 8 * q);
        const int Jq = wp::shfl(Jg, 8 * q);
        const int s0 = (lane & 16) ? (int)(sq >> 16) : (int)(sq & 3u);
        const Walked wk = walk_batch<true>(P, R, Jq, reinterpret_cast<const uint32_t *>(tbq), s0, SlabMode{9, RG_B, RG_NS, 1, 8 * q});
        if (wp::ballot((wk.err & 4) != 0)) passmask &= ~(1u << q);       // cannot happen when the bound holds; full matrix then
        else {
            Q.wk.ops[q][lane] = wk.ops;
            if ((lane & 15) == 0) { Q.wk.n[q][lane >> 4] = wk.n; Q.wk.err[q][lane >> 4] = wk.err; }
        }
    }
    wp::sync();
    if (lane == 0) {
        wp::addg(&P.wb->pair_items, 4);
        wp::addg(&P.wb->ring_kept, 2 * wp::popc(passmask));       // in reads (the host reports pairs)
        wp::addg(&P.wb->ring_sent, 2 * (4 - wp::popc(passmask)));
    }
#pragma unroll 1
    for (int q = 0; q < 4; q++) {
        const int64_t rdA = P.pair_order ? P.pair_order[2 * (first + q)] : 2 * (first + q);
        const int64_t rdB = P.pair_order ? P.pair_order[2 * (first + q) + 1] : 2 * (first + q) + 1;
        RingCtx rc; rc.ops = Q.wk.ops[q]; rc.n = Q.wk.n[q]; rc.err = Q.wk.err[q]; rc.modes = (int)((modes >> (4 * q)) & 15u);
        rc.ref_stride = 0; rc.refmask = 1u;
        process_pair<true>(P, S, staged_prof, rdA, rdB, warp_slot, ((passmask >> q) & 1u) ? &rc : nullptr, P.phase_sync != 0);
        wp::sync();
    }
}

// Ring-banded path when every read is tried against several references (HDR mode, 2..RG_MAX_REFS amplicons): the four pairs'
// combined codes are built once (a pair qualifies only if every reference's seed test picks the same single strand), then
// each reference in turn runs dp_ring over the same codes and its tracebacks, leaving the walked op streams in global
// scratch (rgops); process_pair picks them up per reference and falls back to the full matrix where the band did not hold.
// Kept apart from process_quad and out of line: folded into one inlined template, three amplicons with a coding sequence
// ran 2 % slower (H100, DESIGN.md section 3).
C2B_DEVNOINL void process_quad_multi(const KParams &P, WarpSmem &S, QuadSmem &Q, const uint32_t *staged_prof, int64_t first, int warp_slot)
{
    const int lane = wp::lane(), g = lane >> 3;
    uint2 *tbq = reinterpret_cast<uint2 *>(P.tbq + (int64_t)warp_slot * P.TS * 64);
    uint64_t *rgo = P.rgops + (int64_t)warp_slot * RG_MAX_REFS * 4 * RG_OPS_STRIDE;
    if (P.phase_sync) wp::grp_sync(P.phase_sync);
    uint32_t okmask = 0, modes = 0;
    int Jg = 0, Jmax = 0;
#pragma unroll 1
    for (int q = 0; q < 4; q++) {
        const int64_t rdA = P.pair_order ? P.pair_order[2 * (first + q)] : 2 * (first + q);
        const int64_t rdB = P.pair_order ? P.pair_order[2 * (first + q) + 1] : 2 * (first + q) + 1;
        const int J = (int)(P.offsets[rdA + 1] - P.offsets[rdA]);
        bool bad = false;
#pragma unroll 1
        for (int x = 0; x < 2; x++) bad |= load_codes(P, P.offsets[x ? rdB : rdA], J, S.fw[x], S.rc[x]);
        wp::sync();
        int mAB = 0; bool agree = true;
#pragma unroll 1
        for (int r = 0; r < P.n_refs; r++) {
            int m = 0;
#pragma unroll 1
            for (int x = 0; x < 2; x++) m |= strand_mode(P, P.refs[r], S.fw[x], J) << (2 * x);
            if (r == 0) mAB = m; else agree = agree && (m == mAB);
        }
        const int mA = mAB & 3, mB = mAB >> 2;
        if (!bad && agree && mA != 2 && mB != 2) {
            const uint8_t *cA = mA ? S.rc[0] : S.fw[0], *cB = mB ? S.rc[1] : S.fw[1];
            for (int p = lane; p < J; p += 32) Q.combo[q][p] = (uint8_t)(cA[p] * P.nq + cB[p]);
            okmask |= 1u << q; modes |= (uint32_t)mAB << (4 * q);
            if (g == q) Jg = J;
            if (J > Jmax) Jmax = J;
        }
        wp::sync();
    }
    if (P.phase_sync) wp::grp_sync(P.phase_sync);
    uint32_t passall = 0;                                   // bit 4k + q: the band held for pair q against reference k
    int npass = 0;
#pragma unroll 1
    for (int k = 0; k < P.n_refs && okmask; k++) {
        const RefDev &R = refdev(P, k);
        const bool staged = (k == 0 && staged_prof != nullptr);
        uint32_t *fin = S.rowins;
        if (staged) dp_ring<true>(P, R, staged_prof, Q.combo[g], Jg, Jmax + R.lstar, tbq, fin);
        else dp_ring<false>(P, R, R.prof2, Q.combo[g], Jg, Jmax + R.lstar, tbq, fin);
        wp::sync();
        const int fl = 3 * ((lane & 24) | (R.lstar & 7));
        const uint32_t cM = Jg > 0 ? fin[fl] : PK_SENT, cX = Jg > 0 ? fin[fl + 1] : PK_SENT, cY = Jg > 0 ? fin[fl + 2] : PK_SENT;
        wp::sync();
        const uint32_t z = wp::max3_2(cM, cY, cX);
        const uint32_t s2 = z & PK_TM;
        const int thr = ring_bound(P, R, Jg) + 512 - P.ge * (R.I + Jg);
        const bool pass = Jg > 0 && (int)((z & 0xffffu) >> 2) > thr && (int)(z >> 18) > thr;
        const uint32_t b = wp::ballot(pass);
        uint32_t passmask = (b & 1u) | ((b >> 7) & 2u) | ((b >> 14) & 4u) | ((b >> 21) & 8u);
#pragma unroll 1
        for (int q = 0; q < 4; q++) {
            if (!((passmask >> q) & 1u)) continue;
            const uint32_t sq = wp::shflu(s2, 8 * q);
            const int Jq = wp::shfl(Jg, 8 * q);
            const int s0 = (lane & 16) ? (int)(sq >> 16) : (int)(sq & 3u);
            const Walked wk = walk_batch<true>(P, R, Jq, reinterpret_cast<const uint32_t *>(tbq), s0, SlabMode{9, RG_B, RG_NS, 1, 8 * q});
            if (wp::ballot((wk.err & 4) != 0)) passmask &= ~(1u << q);
            else {
                uint64_t *o = rgo + (int64_t)(k * 4 + q) * RG_OPS_STRIDE;
                o[lane] = wk.ops;
                if ((lane & 15) == 0) o[32 + (lane >> 4)] = (uint64_t)(uint32_t)wk.n | ((uint64_t)(uint32_t)wk.err << 32);
            }
        }
        passall |= passmask << (4 * k);
        npass += wp::popc(passmask);
        wp::sync();
    }
    if (P.phase_sync) wp::grp_sync(P.phase_sync);
    if (lane == 0) {
        wp::addg(&P.wb->pair_items, 4);
        wp::addg(&P.wb->ring_kept, 2 * npass);
        wp::addg(&P.wb->ring_sent, 2 * (4 * P.n_refs - npass));
    }
#pragma unroll 1
    for (int q = 0; q < 4; q++) {
        const int64_t rdA = P.pair_order ? P.pair_order[2 * (first + q)] : 2 * (first + q);
        const int64_t rdB = P.pair_order ? P.pair_order[2 * (first + q) + 1] : 2 * (first + q) + 1;
        RingCtx rc; rc.ops = rgo + (int64_t)q * RG_OPS_STRIDE; rc.n = nullptr; rc.err = nullptr;
        rc.modes = (int)((modes >> (4 * q)) & 15u); rc.ref_stride = 4 * RG_OPS_STRIDE; rc.refmask = 0;
        for (int k = 0; k < P.n_refs; k++) rc.refmask |= ((passall >> (4 * k + q)) & 1u) << k;
        process_pair<false>(P, S, staged_prof, rdA, rdB, warp_slot, ((okmask >> q) & 1u) ? &rc : nullptr, P.phase_sync != 0);
        wp::sync();
    }
}

// Work group wq = work items 4wq..4wq+3 (reads 8wq..8wq+7): four pairs through the ring-banded path when all of them
// qualify, otherwise item by item.
template <bool ONE>
C2B_DEV void process_group(const KParams &P, WarpSmem &S, QuadSmem &Q, const uint32_t *staged_prof, int64_t wq, int warp_slot)
{
    const int lane = wp::lane();
    const int64_t first = 4 * wq;
    const bool multi = !ONE && P.ref_id == nullptr && P.n_refs > 1;
    bool quad = !P.forced_ops && !(P.flags & (C2B_F_NO_PAIRING | C2B_F_NO_RING)) && P.tbq != nullptr &&
                2 * first + 7 < nreads(P) && (!multi || (P.n_refs <= RG_MAX_REFS && P.rgops != nullptr));
    if (quad) {
        const int x = lane & 7;
        const int64_t rd = P.pair_order ? P.pair_order[2 * first + x] : 2 * first + x;
        const int Jx = (int)(P.offsets[rd + 1] - P.offsets[rd]);
        const int rx = P.ref_id ? P.ref_id[rd] : 0;
        const int r0 = wp::shfl(rx, 0);
        const int Jn = wp::shfl_xor(Jx, 1);                 // unconditional: every lane takes part in the exchange
        bool ok = rx == r0 && Jx == Jn && Jx >= 1 && Jx <= RG_COMBO && Jx + 32 <= P.TS;
        const int k0 = multi ? 0 : r0, k1 = multi ? P.n_refs : r0 + 1;
        for (int k = k0; k < k1; k++) {                     // every reference the reads are tried against must admit the band
            const RefDev &R = refdev(P, k);
            ok = ok && R.rg_ok && Jx <= R.pk_maxJ && R.I + Jx <= PK_MAX_ALN && Jx - R.I <= RG_MAXD && R.I - Jx <= RG_MAXD;
        }
        quad = wp::ballot(ok) == 0xffffffffu;
    }
    if (!ONE && quad && multi) process_quad_multi(P, S, Q, staged_prof, first, warp_slot);
    else if (quad) process_quad(P, S, Q, staged_prof, first, warp_slot);
    else {
#pragma unroll 1
        for (int q = 0; q < 4; q++)
            if (2 * (first + q) < nreads(P)) { process_item<ONE>(P, S, staged_prof, first + q, warp_slot); wp::sync(); }
        if (P.phase_sync) {                                 // keep the CTA's barrier count per group the same on every path
#pragma unroll 1
            for (int b = group_phases(P); b > 0; b--) wp::grp_sync(P.phase_sync);
        }
    }
}

// The general kernel's loop over the ALIGN kernel's left-over list (P.pair_order, *P.n_dev entries): one pair per hand-out (a
// warp that drew four hard pairs in a row was the critical path of the whole launch).  `warp` names the warp's scratch slabs.
template <bool ONE>
C2B_DEV void general_list_loop(const KParams &P, WarpSmem &S, const uint32_t *staged_prof, int warp)
{
    const unsigned total = (unsigned)((nreads(P) + 1) / 2);
    for (;;) {
        unsigned w = 0;
        if (wp::lane() == 0) w = (unsigned)wp::fetch_work(P.work_counter);
        w = (unsigned)wp::shfl((int)w, 0);
        if (w >= total) break;
        process_item<ONE>(P, S, staged_prof, (int64_t)w, warp);
        wp::sync();
    }
}

}  // namespace c2b
