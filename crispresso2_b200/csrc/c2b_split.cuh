// c2b_split.cuh -- the hot path as two lean kernels (r02): ALIGN (ring-banded DP + traceback -> op streams in HBM) and
// CLASSIFY (op streams -> aligned strings, find_indels_substitutions, per-read quantification), with the general kernel
// of c2b_core.cuh (c2b_align_classify_kernel: full-matrix paths, any length, --coding_seq, forced op streams) run
// afterwards over the pairs the ALIGN kernel could not prove exact in the band.
//
// Why: the one-kernel form carried 80 KB of hot per-read code against a 32 KB instruction cache and kept its warps in step
// with 23 named barriers per work group (issue slots idle half the time).  Split, every kernel's
// loop fits the cache, no warp waits for another, and the classification is re-formulated in COLUMN space: one alignment
// column per lane, 32 columns per step, reference / read indices from two ballots (no shared-memory scatter, no second
// row-space scan, no per-lane serial loop over 32 columns).
//
//   align_group    reference: CRISPResso2/CRISPResso2Align.pyx:142-421 (DP + traceback), CRISPRessoCORE.py:656-687 (strands)
//   colscan0       reference: Align.pyx:338-434 (the two aligned strings, matchCount), CRISPRessoCORE.py:729-733 (irregular ends)
//   colscan1       reference: CRISPRessoCOREResources.pyx:68-187 + the per-read body of CRISPRessoCORE.py:3989-4115
//   classify_read  reference: CRISPRessoCORE.py:690-798 (best reference, classification), :4195-4272 (HDR re-projection)
#pragma once
#include "c2b_core.cuh"

namespace c2b {

constexpr uint32_t GM_NONE = 0, GM_ALIGNED = 1;        // gmeta state: 0 = not aligned by the ALIGN kernel (general kernel's job)

C2B_DEV uint32_t gmeta_pack(int n, int strand, uint32_t state) { return (uint32_t)n | ((uint32_t)strand << 16) | (state << 24); }

struct ASmem {                                         // ALIGN kernel, per warp
    uint8_t fw[2][RG_COMBO], rc[2][RG_COMBO];          // the two reads of the pair being prepared, as alphabet codes
    uint8_t combo[8][RG_COMBO];                        // base-pair codes of the pairs (four; eight in the narrow first tier)
    uint32_t fin[96];                                  // M, X, Y of cell (I, J) per lane
    uint8_t lut[256];                                  // ASCII -> alphabet code (copy of P.lut: the per-base lookups of load_codes_a
                                                       // waited on global memory, 2.9 % of the tier-1 stall samples at r02k)
};

C2B_DEV void asmem_init(const KParams &P, ASmem &S)
{
    const int lane = wp::lane();
    for (int k = lane; k < 256; k += 32) S.lut[k] = P.lut[k];
    wp::sync();
}

C2B_DEV int64_t read_at(const KParams &P, int64_t idx) { return P.pair_order ? (int64_t)P.pair_order[idx] : idx; }

C2B_DEV void leftover_pair(const KParams &P, int64_t rdA, int64_t rdB)
{
    if (wp::lane() == 0) {
        const unsigned long long pos = wp::fetch_add(&P.wb->launch.left_n, 2ull);
        P.left[pos] = (int32_t)rdA; P.left[pos + 1] = (int32_t)rdB;
    }
}

C2B_DEV void leftover_one(const KParams &P, int64_t rd)
{
    if (wp::lane() == 0) { const unsigned long long pos = wp::fetch_add(&P.wb->launch.left_n, 1ull); P.left[pos] = (int32_t)rd; }
}

// read (its J bytes at src) -> alphabet codes for reads of at most RG_COMBO symbols; true if a symbol is outside the alphabet
C2B_DEV bool load_codes_a(const KParams &P, const uint8_t *lut, const uint8_t *src, int J, uint8_t *fw, uint8_t *rc)
{
    const int lane = wp::lane();
    bool bad = false;
    for (int base = 0; base < J; base += 128) {
        uint8_t ch[4];
#pragma unroll
        for (int e = 0; e < 4; e++) { const int p = base + lane + 32 * e; ch[e] = p < J ? src[p] : (uint8_t)P.alpha[0]; }
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int p = base + lane + 32 * e;
            int code = lut[ch[e]];
            if (code == 255) { bad = true; code = 0; }
            if (p < J) { fw[p] = (uint8_t)code; rc[J - 1 - p] = P.comp[code]; }
        }
    }
    return wp::ballot(bad) != 0;
}

// Four tracebacks of one ring-banded DP at once.  walk_batch (c2b_core.cuh) is a chain of dependent L2 round trips -- one
// slab gather per run of equal ops -- and four of them in sequence cost as much wall time as the DP itself (r02b: the ALIGN
// kernel's issue slots were idle half the time).  Here every iteration issues the gathers of all four pairs before it
// consumes any, so the four latencies overlap; the per-pair logic is walk_batch<true>'s for a ring slab, verbatim.
// RL / q0 / NP: ring size of the DP that filled the slab (8 or 4 lanes), first pair and number of pairs walked (interleaved) by this call.
template <int RL = 8, int NP = 4>
C2B_DEV void walk_ring4(const KParams &P, const RefDev &R, const int *Jq, const uint2 *__restrict__ tb2, const int *s0, uint32_t mask,
                        Walked *out, const int q0 = 0)
{
    constexpr int NS = 9 * RL, B = 4 * RL;
    const int lane = wp::lane();
    const int hl = lane & 15, hb = lane & 16;
    const int TS = P.TS;
    int i[NP], j[NP], s[NP], n[NP], err[NP];
    uint32_t acc[NP], lo[NP], hi[NP];
#pragma unroll
    for (int q = 0; q < NP; q++) {
        const bool on = (mask >> q) & 1u;
        i[q] = on ? R.I : 0; j[q] = on ? Jq[q] : 0; s[q] = s0[q]; n[q] = 0; err[q] = 0; acc[q] = 0; lo[q] = hi[q] = ~0u;
    }
    // append `cnt` (<= 32) copies of op to pair q's stream; acc holds the (n & 15) newest ops in its top bits
#define C2B_PUSH4(q, op_, cnt_) do { int cnt = (cnt_); const uint32_t pat = (uint32_t)(op_) * 0x55555555u;                          \
        while (cnt > 0) { const int room = 16 - (n[q] & 15); const int c = cnt < room ? cnt : room;                                  \
            acc[q] = (uint32_t)((((uint64_t)pat << 32) | acc[q]) >> (2 * c)); n[q] += c; cnt -= c;                                   \
            if ((n[q] & 15) == 0) { const int ix = (n[q] >> 4) - 1; if (hl == (ix >> 1)) { if (ix & 1) hi[q] = acc[q]; else lo[q] = acc[q]; } } } } while (0)
    for (;;) {
        uint2 w2[NP]; bool valid[NP], inband[NP]; int sh[NP];
        bool anyact = false;
#pragma unroll
        for (int q = 0; q < NP; q++) {
            const bool active = i[q] > 0 && j[q] > 0;
            anyact |= active;
            const int di = (s[q] != OP_I), dj = (s[q] != OP_J);
            const int ci = i[q] - hl * di, cj = j[q] - hl * dj;
            valid[q] = active && ci >= 1 && cj >= 1;
            inband[q] = valid[q];
            w2[q] = make_uint2(0u, 0u); sh[q] = 0;
            if (valid[q]) {
                const int r = ci - 1, l = (r >> 3) & 31;
                const int slot = cj + l - 9 * l + B;
                inband[q] = (unsigned)slot < (unsigned)NS;
                sh[q] = 2 * (7 - (r & 7));
                if (inband[q]) w2[q] = wp::ldcg2(tb2 + (int64_t)(RL * (q0 + q) + (l & (RL - 1))) * TS + cj + l);
            }
        }
        if (!wp::ballot(anyact)) break;
#pragma unroll
        for (int q = 0; q < NP; q++) {
            const bool active = i[q] > 0 && j[q] > 0;
            const uint32_t w = hb ? ((w2[q].x & 0xffff0000u) | (w2[q].y >> 16)) : ((w2[q].x << 16) | (w2[q].y & 0xffffu));
            const uint32_t v = (valid[q] && inband[q]) ? (w >> sh[q]) : 0u;
            const int tag = (int)((v >> 16) & 3u);
            const bool cont = valid[q] && (s[q] == OP_M ? tag == OP_M : (v & (uint32_t)s[q]) != 0u);
            const uint32_t bc = (wp::ballot(cont) >> hb) & 0xffffu, bv = (wp::ballot(valid[q]) >> hb) & 0xffffu;
            const uint32_t bo = (wp::ballot(valid[q] && !inband[q]) >> hb) & 0xffffu;
            int nvalid = wp::popc(bv);
            if (bo) { const int fo = wp::ffs(bo) - 1; if (fo < nvalid) nvalid = fo; }
            const bool miss = active && nvalid == 0;
            int f = wp::ffs(~bc) - 1;
            if (f < 0 || f > nvalid) f = nvalid;
            const bool brk = f < nvalid;
            const int run = brk ? f + 1 : nvalid;
            const int tagf = wp::shfl(tag, hb + (f < 16 ? f : 15));
            if (miss) { err[q] |= 4; i[q] = 0; j[q] = 0; }
            else if (active) {
                const int di = (s[q] != OP_I), dj = (s[q] != OP_J);
                const int news = brk ? (s[q] == OP_M ? tagf : OP_M) : s[q];
                C2B_PUSH4(q, s[q], run);
                i[q] -= run * di; j[q] -= run * dj;
                err[q] |= (news == 3);
                s[q] = news;
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NP; q++) {
        if (j[q] > 0 && s[q] != OP_I) err[q] |= 1;              // row 0 / column 0 can only be left along their own border
        if (i[q] > 0 && s[q] != OP_J) err[q] |= 1;
        while (j[q] > 0) { const int c = j[q] < 32 ? j[q] : 32; C2B_PUSH4(q, OP_I, c); j[q] -= c; }
        while (i[q] > 0) { const int c = i[q] < 32 ? i[q] : 32; C2B_PUSH4(q, OP_J, c); i[q] -= c; }
        if (n[q] & 15) {
            const int ix = n[q] >> 4, used = 2 * (n[q] & 15);
            const uint32_t a = (acc[q] >> (32 - used)) | (~0u << used);
            if (hl == (ix >> 1)) { if (ix & 1) hi[q] = a; else lo[q] = a; }
        }
        out[q].ops = (uint64_t)lo[q] | ((uint64_t)hi[q] << 32); out[q].ops2 = ~0ull; out[q].n = n[q]; out[q].err = err[q];
    }
#undef C2B_PUSH4
}

// matchCount (Align.pyx:338-421: columns where both strings hold the same character; N over N counts) of the alignment a pair
// walk left in this half-warp's lanes: lane hl holds columns 32 hl .. of `ops` and 512 + 32 hl .. of `ops2`, counted from the
// right end.  codes: the read as alphabet codes in the strand that was aligned.  All 32 lanes call; the result is per half.
C2B_DEV int match_count_half(const KParams &P, const RefDev &R, const uint8_t *codes, int J, const Walked &wk)
{
    const int hl = wp::lane() & 15;
    const uint64_t lo = 0x5555555555555555ull;
    int base_i = R.I, base_j = J, match = 0;
#pragma unroll 1
    for (int word = 0; word < 2; word++) {
        const uint64_t ops = word ? wk.ops2 : wk.ops;
        const int ci = 32 - wp::popcll((ops >> 1) & lo);     // ops consuming a reference base (M, J); OP_NONE counts for neither
        const int cj = 32 - wp::popcll(ops & lo);            // ops consuming a read base (M, I)
        int pk = (ci << 16) | cj;
#pragma unroll
        for (int d = 1; d < 16; d <<= 1) { const int v = wp::shfl_up(pk, d); if (hl >= d) pk += v; }
        const int tot = wp::shfl(pk, (wp::lane() & 16) | 15);
        pk -= (ci << 16) | cj;                               // exclusive prefix inside the half-warp
        int i = base_i - (pk >> 16), j = base_j - (pk & 0xffff);
        uint64_t rest = ops;
#pragma unroll 4
        for (int e = 0; e < 32; e++) {
            const int op = (int)rest & 3;
            rest >>= 2;
            if (op == OP_NONE) continue;
            if (op == OP_M && (uint32_t)P.alpha[codes[j - 1]] == (uint32_t)R.asc[i - 1]) match++;
            i -= (op != OP_I); j -= (op != OP_J);
        }
        base_i -= tot >> 16; base_j -= tot & 0xffff;
    }
#pragma unroll
    for (int d = 8; d >= 1; d >>= 1) match += wp::shfl_xor(match, d);
    return match;
}

// ---------------------------------------------------------------------------------------------------- ALIGN
// Work group wq = reads 8wq..8wq+7 (four pairs).  Eligible groups (equal lengths per pair, every candidate reference admits
// the band) run the ring-banded DP once per candidate reference and walk the four tracebacks; a pair whose two scores beat
// the out-of-band bound for EVERY candidate reference leaves its op streams in P.gops and is marked GM_ALIGNED; every other
// pair goes to the left-over list of the general kernel.
C2B_DEV void align_group(const KParams &P, ASmem &S, const uint32_t *staged_prof, int64_t wq, int warp_slot)
{
    const int lane = wp::lane(), g = lane >> 3;
    const int64_t first = 4 * wq;
    const bool multi = P.ref_id == nullptr && P.n_refs > 1;
    // A group is taken here when its four pairs admit the packed 16-bit DP against every candidate reference (equal lengths
    // within a pair, lengths inside the proven 16-bit range); per reference the ring-banded DP is tried when the band can hold
    // the alignment (read length within RG_MAXD of the amplicon's, monotone bound), the full matrix otherwise.
    bool quad = (P.tbq != nullptr || P.tb != nullptr) && 2 * first + 7 < nreads(P) && (!multi || P.n_refs <= RG_MAX_REFS);
    int r0 = 0;
    uint32_t ringmask = 0;                                   // bit k - k0: the ring-banded DP is admissible for reference k
    if (quad) {
        const int x = lane & 7;
        const int64_t rd = read_at(P, 2 * first + x);
        const int Jx = (int)(P.offsets[rd + 1] - P.offsets[rd]);
        const int rx = P.ref_id ? P.ref_id[rd] : 0;
        r0 = wp::shfl(rx, 0);
        const int Jn = wp::shfl_xor(Jx, 1);
        bool ok = rx == r0 && Jx == Jn && Jx >= 1 && Jx <= RG_COMBO && Jx + 32 <= P.TS;
        const int k0 = multi ? 0 : r0, k1 = multi ? P.n_refs : r0 + 1;
        for (int k = k0; k < k1; k++) {
            const RefDev &R = refdev(P, k);
            ok = ok && !R.coding && Jx <= R.pk_maxJ;
            const bool rk = P.tbq != nullptr && R.rg_ok && R.I + Jx <= PK_MAX_ALN && Jx - R.I <= RG_MAXD && R.I - Jx <= RG_MAXD;
            if (wp::ballot(rk) == 0xffffffffu) ringmask |= 1u << (k - k0);
        }
        quad = wp::ballot(ok) == 0xffffffffu;
        if (!P.tb && ringmask != (k1 - k0 >= 32 ? 0xffffffffu : (1u << (k1 - k0)) - 1u)) quad = false;    // no full-matrix scratch
    }
    if (!quad) {
#pragma unroll 1
        for (int q = 0; q < 4; q++) {
            if (2 * (first + q) >= nreads(P)) break;
            const int64_t rdA = read_at(P, 2 * (first + q));
            // the list mixes pairs and single reads, and the general kernel takes its entries two at a time: the odd last read
            // goes on it ONCE (an (rdA, rdA) entry could be split over two work items and be counted twice)
            if (2 * (first + q) + 1 < nreads(P)) leftover_pair(P, rdA, read_at(P, 2 * (first + q) + 1));
            else leftover_one(P, rdA);
        }
        return;
    }
    const int k0 = multi ? 0 : r0, k1 = multi ? P.n_refs : r0 + 1;
    uint2 *tbq = P.tbq ? reinterpret_cast<uint2 *>(P.tbq + (int64_t)warp_slot * P.TS * 64) : nullptr;
    uint32_t okmask = 0, modes = 0;
    // both2[k - k0]: reads (bit 2q + h) that reference k's seed test wants aligned on both strands.  The seed tests of the
    // candidate references may disagree (r02y: 8 % of the HDR bench reads miss the seeds of ONE amplicon; their pairs used to go
    // to the general kernel, which then cost 44 % of the HDR step): the strand a read rides the packed DP on is the first
    // reference's choice, a reference that wants both strands gets its own both-strand alignment below, and only a forward /
    // reverse-complement conflict between references still sends the pair on.
    uint32_t both2[RG_MAX_REFS] = {0, 0, 0, 0};
    int Jg = 0, Jmax = 0;
#pragma unroll 1
    for (int q = 0; q < 4; q++) {
        const int64_t rdA = read_at(P, 2 * (first + q)), rdB = read_at(P, 2 * (first + q) + 1);
        const int J = (int)(P.offsets[rdA + 1] - P.offsets[rdA]);
        bool bad = false;
#pragma unroll 1
        for (int x = 0; x < 2; x++) bad |= load_codes_a(P, S.lut, P.reads + P.offsets[x ? rdB : rdA], J, S.fw[x], S.rc[x]);
        wp::sync();
        int mAB = 0; bool agree = true;
        uint32_t bothq[RG_MAX_REFS] = {0, 0, 0, 0};
#pragma unroll 1
        for (int k = k0; k < k1; k++) {
            int m = 0;
#pragma unroll 1
            for (int x = 0; x < 2; x++) m |= strand_mode(P, refdev(P, k), S.fw[x], J) << (2 * x);
            if (k == k0) mAB = m;
#pragma unroll
            for (int x = 0; x < 2; x++) {
                const int mk = (m >> (2 * x)) & 3, m0 = (mAB >> (2 * x)) & 3;
                if (mk == 2) bothq[(k - k0) & (RG_MAX_REFS - 1)] |= 1u << x;        // this reference: both strands, whatever the ride
                else if (mk != (m0 == 2 ? 0 : m0)) agree = false;                    // forward here, reverse complement there
            }
        }
        const int mA = mAB & 3, mB = mAB >> 2;
        if (!bad && agree) {
            // a read whose seed test calls for both strands (mode 2) rides along on its forward strand -- its half of the ring
            // result is ignored for that reference -- and is aligned on both strands over the full matrix below (r02d: such a read
            // sent its whole pair to the general kernel: 0.8 % of the reads, a twentieth of the batch's time)
            const uint8_t *cA = mA == 1 ? S.rc[0] : S.fw[0], *cB = mB == 1 ? S.rc[1] : S.fw[1];
            for (int p = lane; p < J; p += 32) S.combo[q][p] = (uint8_t)(cA[p] * P.nq + cB[p]);
            okmask |= 1u << q; modes |= (uint32_t)mAB << (4 * q);
#pragma unroll
            for (int kk = 0; kk < RG_MAX_REFS; kk++) both2[kk] |= bothq[kk] << (2 * q);
            if (g == q) Jg = J;
            if (J > Jmax) Jmax = J;
        }
        wp::sync();
    }
    // reads (bit 2q + h: read h of pair q) whose band held for every reference so far.  The two halves of a packed value
    // are independent DPs, so a pair may keep one read and send only the other to the general kernel (r02b: per pair,
    // which doubled the left-over list).
    uint32_t good2 = 0;
#pragma unroll
    for (int q = 0; q < 4; q++) if ((okmask >> q) & 1u) good2 |= 3u << (2 * q);
    if (!P.tb) {                                            // no full-matrix scratch: general kernel
#pragma unroll
        for (int kk = 0; kk < RG_MAX_REFS; kk++) { good2 &= ~both2[kk]; both2[kk] = 0; }
    }
    int npass = 0, ntried = 0, nboth = 0;
#pragma unroll 1
    for (int k = k0; k < k1 && good2; k++) {
        const RefDev &R = refdev(P, k);
        const uint32_t bothk = both2[(k - k0) & (RG_MAX_REFS - 1)];
        const uint32_t ring2 = good2 & ~bothk;              // reads whose ring result counts for this reference
        nboth += wp::popc(bothk & good2);
        const bool staged = (k == 0 && staged_prof != nullptr);
        uint32_t pass2 = 0;
        if (((ringmask >> (k - k0)) & 1u) && ring2) {
        if (staged) dp_ring<true>(P, R, staged_prof, S.combo[g], Jg, Jmax + R.lstar, tbq, S.fin);
        else dp_ring<false>(P, R, R.prof2, S.combo[g], Jg, Jmax + R.lstar, tbq, S.fin);
        wp::sync();
        const int fl = 3 * ((lane & 24) | (R.lstar & 7));
        const uint32_t cM = Jg > 0 ? S.fin[fl] : PK_SENT, cX = Jg > 0 ? S.fin[fl + 1] : PK_SENT, cY = Jg > 0 ? S.fin[fl + 2] : PK_SENT;
        wp::sync();
        const uint32_t z = wp::max3_2(cM, cY, cX);
        const uint32_t s2 = z & PK_TM;
        // biased value = 4*(score + beta*(I+J) + 512) + tag: a read must beat the out-of-band bound (ring_bound)
        const int thr = ring_bound(P, R, Jg) + 512 - P.ge * (R.I + Jg);
        const bool passA = Jg > 0 && (int)((z & 0xffffu) >> 2) > thr, passB = Jg > 0 && (int)(z >> 18) > thr;
        const uint32_t bA = wp::ballot(passA), bB = wp::ballot(passB);
#pragma unroll
        for (int q = 0; q < 4; q++) pass2 |= (((bA >> (8 * q)) & 1u) | (((bB >> (8 * q)) & 1u) << 1)) << (2 * q);
        pass2 &= ring2;
        ntried += wp::popc(ring2);
        {
            int Jq[4], s0[4];
            Walked wk4[4];
            uint32_t walkmask = 0;
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const uint32_t sq = wp::shflu(s2, 8 * q);
                Jq[q] = wp::shfl(Jg, 8 * q);
                s0[q] = (lane & 16) ? (int)(sq >> 16) : (int)(sq & 3u);
                if ((pass2 >> (2 * q)) & 3u) walkmask |= 1u << q;
            }
            walk_ring4(P, R, Jq, tbq, s0, walkmask, wk4);
#pragma unroll
            for (int q = 0; q < 4; q++) {
                if (!((walkmask >> q) & 1u)) continue;
                const Walked &wk = wk4[q];
                const uint32_t eb = wp::ballot(wk.err != 0);             // cannot happen when the bound holds; general kernel then
                if (eb & 0xffffu) pass2 &= ~(1u << (2 * q));
                if (eb >> 16) pass2 &= ~(2u << (2 * q));
                const int h = lane >> 4, hl = lane & 15;
                if (!((pass2 >> (2 * q + h)) & 1u)) continue;
                const int64_t rd = read_at(P, 2 * (first + q) + h);
                const int64_t slot = oslot(P, rd, k);
                if (hl < P.NW) P.gops[slot * P.NW + hl] = wk.ops;
                if (hl == 0) {
                    const int mode = (int)((modes >> (4 * q + 2 * h)) & 3u);
                    P.gmeta[slot] = gmeta_pack(wk.n, mode == 1, GM_NONE);        // state is set below, once every reference passed
                }
            }
        }
        npass += wp::popc(pass2);
        } else ntried += wp::popc(ring2);
        // Full-matrix DPs (align_pair, the packed path of c2b_core.cuh), here and now, for what the ring did not settle for this
        // reference: (job 0) pairs with a read the ring could not prove exact; (jobs 1, 2) a read that needs both strands,
        // packed with ITSELF -- forward strand in the low halves, reverse complement in the high ones -- the better identity
        // wins, the reverse complement only if strictly better (CRISPRessoCORE.py:678-687).  r02b sent all of these to the
        // general kernel, whose launch then spent its time on 0.8 % of the reads: the latency of single pairs through its whole
        // per-read path; inside this persistent kernel the same DPs hide among the other warps' work.
        const uint32_t failed = ring2 & ~pass2;
        if ((failed | (bothk & good2)) && P.tb) {
            uint2 *tb2 = reinterpret_cast<uint2 *>(P.tb + (int64_t)warp_slot * P.tb_words_per_warp);
            int32_t *bnd = P.bnd + (int64_t)warp_slot * P.bnd_words_per_warp;
            const int h = lane >> 4, hl = lane & 15;
#pragma unroll 1
            for (int job = 0; job < 16; job++) {
                const int q = job >> 2, kind = job & 3;              // kind 0: pair q; 1 / 2: read A / B of pair q on both strands
                if (kind == 3) continue;
                const uint32_t fq = (failed >> (2 * q)) & 3u;
                const uint32_t bq = ((bothk & good2) >> (2 * q)) & 3u;
                if (kind == 0 ? fq == 0 : !((bq >> (kind - 1)) & 1u)) continue;
                const int Jp = wp::shfl(Jg, 8 * q);
                const uint8_t *combo = S.combo[q];
                wp::sync();
                if (kind) {
                    const int64_t rdx = read_at(P, 2 * (first + q) + (kind - 1));
                    load_codes_a(P, S.lut, P.reads + P.offsets[rdx], Jp, S.fw[0], S.rc[0]);
                    wp::sync();
                    for (int p = lane; p < Jp; p += 32) S.fw[1][p] = (uint8_t)(S.fw[0][p] * P.nq + S.rc[0][p]);
                    combo = S.fw[1];
                    wp::sync();
                }
                const Walked wk = align_pair(P, R, staged ? staged_prof : R.prof2, staged, combo, Jp, tb2, nullptr, bnd);
                const uint32_t eb = wp::ballot(wk.err != 0);             // the reference's undefined zone: general kernel
                if (kind == 0) {
                    const bool mine = ((fq >> h) & 1u) && !((h ? (eb >> 16) : (eb & 0xffffu)));
                    if (mine) {
                        const int64_t rd = read_at(P, 2 * (first + q) + h);
                        const int64_t slot = oslot(P, rd, k);
                        if (hl < P.NW) P.gops[slot * P.NW + hl] = wk.ops;
                        if (hl + 16 < P.NW) P.gops[slot * P.NW + 16 + hl] = wk.ops2;
                        if (hl == 0) P.gmeta[slot] = gmeta_pack(wk.n, (int)((modes >> (4 * q + 2 * h)) & 3u) == 1, GM_NONE);
                    }
                    const uint32_t mb = wp::ballot(mine);
                    if (mb & 0xffffu) pass2 |= 1u << (2 * q);
                    if (mb >> 16) pass2 |= 2u << (2 * q);
                } else {
                    const int nm = match_count_half(P, R, h ? S.rc[0] : S.fw[0], Jp, wk);
                    const int sc = score_milli(nm, wk.n > 0 ? wk.n : 1);
                    const int sc_fw = wp::shfl(sc, 0), sc_rc = wp::shfl(sc, 16);
                    const int pick = sc_rc > sc_fw ? 1 : 0;
                    const uint32_t bit = 1u << (2 * q + kind - 1);
                    if (eb) good2 &= ~bit;                                   // either strand undefined: the general kernel decides
                    else if (h == pick) {
                        const int64_t rd = read_at(P, 2 * (first + q) + (kind - 1));
                        const int64_t slot = oslot(P, rd, k);
                        if (hl < P.NW) P.gops[slot * P.NW + hl] = wk.ops;
                        if (hl + 16 < P.NW) P.gops[slot * P.NW + 16 + hl] = wk.ops2;
                        if (hl == 0) P.gmeta[slot] = gmeta_pack(wk.n, pick, GM_NONE);
                    }
                }
            }
        }
        pass2 |= bothk & good2;                                              // both-strand reads: settled above (or dropped from good2)
        good2 &= pass2;
        wp::sync();
    }
#ifndef C2B_EMU
    // the slab is dead now: drop its lines from L2 instead of writing them back to HBM (10 KB per read otherwise)
    if (tbq && ringmask) {
        const char *base = reinterpret_cast<const char *>(tbq);
        const int64_t bytes = (int64_t)P.TS * 64 * 4;
        for (int64_t o = (int64_t)lane * 128; o < bytes; o += 32 * 128)
            asm volatile("discard.global.L2 [%0], 128;" ::"l"(base + o) : "memory");
    }
#endif
    if (lane == 0) {                                         // path statistics, in reads (the host reports pairs)
        wp::addg(&P.wb->align_settled, wp::popc(good2));
        wp::addg(&P.wb->ring_kept, npass);
        wp::addg(&P.wb->ring_sent, ntried - npass + nboth + 2 * (k1 - k0) * (4 - wp::popc(okmask)));
    }
#pragma unroll 1
    for (int q = 0; q < 4; q++) {
        const int64_t rdA = read_at(P, 2 * (first + q)), rdB = read_at(P, 2 * (first + q) + 1);
        const uint32_t gq = (good2 >> (2 * q)) & 3u;
        if (gq) {
            const int64_t rd = (lane & 1) ? rdB : rdA;
            const int k = k0 + (lane >> 1);
            if (k < k1 && ((gq >> (lane & 1)) & 1u)) { const int64_t slot = oslot(P, rd, k); P.gmeta[slot] = (P.gmeta[slot] & 0x00ffffffu) | (GM_ALIGNED << 24); }
        }
        if (gq == 0) leftover_pair(P, rdA, rdB);
        else if (gq != 3u) leftover_one(P, gq == 1u ? rdB : rdA);
    }
}

// ---------------------------------------------------------------------------------------- ALIGN, narrow first tier (r02i)
// Sixteen reads (eight pairs) per warp in ONE ring-banded pass: rings of four lanes, band of 36 slots (cells with column - row
// in about [-17, +11]).  Same DP, same exactness argument with the narrower band's bound (ring_bound(.., 17, 11)): a read
// whose banded score beats it -- every read within ~10 substitutions of the amplicon, deletions up to ~8 bp, insertions up to
// ~9 bp: 84 % of the bench reads -- has its exact full-matrix traceback at half the cost per read.  Every other read goes,
// alone, on the tier-2 list (P.left2), which a second launch of this kernel works through in groups of eight with the
// 72-slot band, the full matrix and the both-strand alignment of align_group.
// Taken only for sixteen consecutive reads of one length and one single candidate reference that admits the ring; returns
// false otherwise (the caller runs align_group on the two groups of eight).
C2B_DEV bool align_narrow16(const KParams &P, ASmem &S, const uint32_t *staged_prof, int64_t w16, int warp_slot)
{
    constexpr int RL = 4, DLO = 4 * RL + 1, DHI = 9 * RL - 4 * RL - 9;
    static_assert(DLO == RN_DLO && DHI == RN_DHI, "the diagonal tier's routing test assumes this band");
    const int lane = wp::lane(), g = lane >> 2;
    const int64_t first = 16 * w16;                         // first read
    if (!P.left2 || P.tbq == nullptr || first + 15 >= nreads(P) || (P.ref_id == nullptr && P.n_refs > 1)) return false;
    int r0, J0;
    {
        const int64_t rd = read_at(P, first + (lane & 15));
        const int Jx = (int)(P.offsets[rd + 1] - P.offsets[rd]);
        const int rx = P.ref_id ? P.ref_id[rd] : 0;
        r0 = wp::shfl(rx, 0); J0 = wp::shfl(Jx, 0);
        const RefDev &R = refdev(P, r0);
        const bool ok = rx == r0 && Jx == J0 && Jx >= 1 && Jx <= RG_COMBO && Jx + 32 <= P.TS && R.rg_ok && !R.coding && Jx <= R.pk_maxJ &&
                        R.I + Jx <= PK_MAX_ALN && Jx - R.I <= RG_MAXD && R.I - Jx <= RG_MAXD;
        if (wp::ballot(ok) != 0xffffffffu) return false;
    }
    const RefDev &R = refdev(P, r0);
    const int J = J0;
    uint2 *tbq = reinterpret_cast<uint2 *>(P.tbq + (int64_t)warp_slot * P.TS * 64);
    uint32_t modes = 0, use2 = 0;                            // use2: reads (bit 2q + h) whose ring result counts
#pragma unroll 1
    for (int q = 0; q < 8; q++) {
        const int64_t rdA = read_at(P, first + 2 * q), rdB = read_at(P, first + 2 * q + 1);
        bool badA = load_codes_a(P, S.lut, P.reads + P.offsets[rdA], J, S.fw[0], S.rc[0]);
        bool badB = load_codes_a(P, S.lut, P.reads + P.offsets[rdB], J, S.fw[1], S.rc[1]);
        wp::sync();
        int m = 0;
#pragma unroll 1
        for (int x = 0; x < 2; x++) m |= strand_mode(P, R, S.fw[x], J) << (2 * x);
        const int mA = m & 3, mB = m >> 2;
        // a read with a symbol outside the alphabet or in need of both strands rides along on its forward strand; tier 2 settles it
        const uint8_t *cA = mA == 1 ? S.rc[0] : S.fw[0], *cB = mB == 1 ? S.rc[1] : S.fw[1];
        for (int p = lane; p < J; p += 32) S.combo[q][p] = (uint8_t)(cA[p] * P.nq + cB[p]);
        modes |= (uint32_t)m << (4 * q);
        if (!badA && mA != 2) use2 |= 1u << (2 * q);
        if (!badB && mB != 2) use2 |= 2u << (2 * q);
        wp::sync();
    }
    const bool staged = (r0 == 0 && staged_prof != nullptr);
    if (staged) dp_ring<true, RL>(P, R, staged_prof, S.combo[g], J, J + R.lstar, tbq, S.fin);
    else dp_ring<false, RL>(P, R, R.prof2, S.combo[g], J, J + R.lstar, tbq, S.fin);
    wp::sync();
    const int fl = 3 * ((lane & ~(RL - 1)) | (R.lstar & (RL - 1)));
    const uint32_t cM = S.fin[fl], cX = S.fin[fl + 1], cY = S.fin[fl + 2];
    wp::sync();
    const uint32_t z = wp::max3_2(cM, cY, cX);
    const uint32_t s2 = z & PK_TM;
    const int thr = ring_bound(P, R, J, DLO, DHI) + 512 - P.ge * (R.I + J);
    const uint32_t bA = wp::ballot((int)((z & 0xffffu) >> 2) > thr), bB = wp::ballot((int)(z >> 18) > thr);
    uint32_t pass2 = 0;
#pragma unroll
    for (int q = 0; q < 8; q++) pass2 |= (((bA >> (RL * q)) & 1u) | (((bB >> (RL * q)) & 1u) << 1)) << (2 * q);
    pass2 &= use2;
    // tracebacks: pairs 0-3, then 4-7, four interleaved at a time (all eight at once was measured slower)
#pragma unroll 1
    for (int half = 0; half < 2; half++) {
        const int q0 = 4 * half;
        int Jq[4], s0[4];
        Walked wk4[4];
        uint32_t walkmask = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t sq = wp::shflu(s2, RL * (q0 + q));
            Jq[q] = J;
            s0[q] = (lane & 16) ? (int)(sq >> 16) : (int)(sq & 3u);
            if ((pass2 >> (2 * (q0 + q))) & 3u) walkmask |= 1u << q;
        }
        if (!walkmask) continue;
        walk_ring4<RL, 4>(P, R, Jq, tbq, s0, walkmask, wk4, q0);
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (!((walkmask >> q) & 1u)) continue;
            const int qq = q0 + q;
            const Walked &wk = wk4[q];
            const uint32_t eb = wp::ballot(wk.err != 0);
            if (eb & 0xffffu) pass2 &= ~(1u << (2 * qq));
            if (eb >> 16) pass2 &= ~(2u << (2 * qq));
            const int h = lane >> 4, hl = lane & 15;
            if (!((pass2 >> (2 * qq + h)) & 1u)) continue;
            const int64_t rd = read_at(P, first + 2 * qq + h);
            const int64_t slot = oslot(P, rd, r0);
            if (hl < P.NW) P.gops[slot * P.NW + hl] = wk.ops;
            if (hl == 0) P.gmeta[slot] = gmeta_pack(wk.n, (int)((modes >> (4 * qq + 2 * h)) & 3u) == 1, GM_ALIGNED);
        }
    }
#ifndef C2B_EMU
    {                                                        // the slab is dead now: drop its lines from L2
        const char *base = reinterpret_cast<const char *>(tbq);
        const int64_t bytes = (int64_t)P.TS * 64 * 4;
        for (int64_t o = (int64_t)lane * 128; o < bytes; o += 32 * 128)
            asm volatile("discard.global.L2 [%0], 128;" ::"l"(base + o) : "memory");
    }
#endif
    // everything the narrow band did not settle: one entry each on the tier-2 list
    const uint32_t rest = 0xffffu & ~pass2;
    if (lane < 16 && ((rest >> lane) & 1u)) {
        const unsigned long long pos = wp::fetch_add(&P.wb->launch.tier2_n, 1ull);
        P.left2[pos] = (int32_t)read_at(P, first + lane);
    }
    if (lane == 0) {
        wp::addg(&P.wb->align_settled, wp::popc(pass2));
        wp::addg(&P.wb->ring_kept, wp::popc(pass2));
        wp::addg(&P.wb->tier2, 16 - wp::popc(pass2));
    }
    return true;
}

// The ALIGN kernel's loop for warp `warp`: persistent, free-running warps pull work from a counter -- units of sixteen reads
// with the narrow first tier (units it does not take run as two ordinary groups of eight), groups of eight without it.  The
// work a warp is likely to get next has its bytes sent towards L2.  The number of warps is read from the grid where it is
// used: passed in as a value it stays live across the DP calls, and the kernel spills more at its 128-register limit.
C2B_DEV void align_loop(const KParams &P, ASmem &S, const uint32_t *staged_prof, int warp)
{
    const int lane = wp::lane();
    asmem_init(P, S);
    const int64_t nrd = nreads(P);
    const unsigned ahead = (unsigned)wp::grid_warps();
    if (P.left2) {
        const unsigned total = (unsigned)((nrd + 15) / 16);
        for (;;) {
            unsigned w = 0;
            if (lane == 0) w = (unsigned)wp::fetch_work(P.work_counter);
            w = (unsigned)wp::shfl((int)w, 0);
            if (w >= total) break;
            if (w + ahead < total) {
                const int64_t g = (int64_t)w + ahead;
                if (!P.pair_order) {
                    const int64_t last = 16 * g + 16 < nrd ? 16 * g + 16 : nrd;
                    const int64_t a = P.offsets[16 * g] + (int64_t)lane * 128;
                    if (a < P.offsets[last]) wp::prefetch_l2(P.reads + a);
                } else {                                        // reads of the diagonal tier's list: two lanes per read
                    const int64_t x = 16 * g + (lane >> 1);
                    if (x < nrd) {
                        const int64_t rd = read_at(P, x);
                        const int64_t b1 = P.offsets[rd + 1];
                        for (int64_t a = (P.offsets[rd] & ~(int64_t)127) + (int64_t)(lane & 1) * 128; a < b1; a += 256)
                            wp::prefetch_l2(P.reads + a);
                    }
                }
            }
            if (!align_narrow16(P, S, staged_prof, (int64_t)w, warp)) {
                align_group(P, S, staged_prof, 2 * (int64_t)w, warp);
                wp::sync();
                if (8 * (2 * (int64_t)w + 1) < nrd) align_group(P, S, staged_prof, 2 * (int64_t)w + 1, warp);
            }
            wp::sync();
        }
        return;
    }
    const unsigned total = (unsigned)((nrd + 7) / 8);
    for (;;) {
        unsigned w = 0;
        if (lane == 0) w = (unsigned)wp::fetch_work(P.work_counter);
        w = (unsigned)wp::shfl((int)w, 0);
        if (w >= total) break;
        if (w + ahead < total && !P.pair_order) {
            const int64_t g = (int64_t)w + ahead;
            const int64_t last = 8 * g + 8 < nrd ? 8 * g + 8 : nrd;
            const int64_t a = P.offsets[8 * g] + (int64_t)lane * 128;
            if (a < P.offsets[last]) wp::prefetch_l2(P.reads + a);
        }
        align_group(P, S, staged_prof, (int64_t)w, warp);
        wp::sync();
    }
}

// ------------------------------------------------------------------------------------------------- CLASSIFY
// One alignment per warp, one column per lane, 32 columns per step, left to right.  Column c (from the left) is op number
// n-1-c of the stream (the walk emits right to left).  With bI / bJ the ballots of the insertion / deletion columns of a
// step, lane l's reference index is i0 + l - popc(bI below l) and its read index j0 + l - popc(bJ below l).
// The read's bytes and its op streams are staged in shared memory by the kernel loop (one coalesced 16-byte load per lane,
// issued one read ahead), so the scans below touch global memory only for the reference tables (L1-resident) and outputs.
constexpr int B_RD_BYTES = 32 * 16;                    // staged window of read bytes (16-byte aligned start)

// Per-warp accumulators of the per-reference scalar counters (RefDev::scal): lane s holds slot s of the reference named in
// `ref`.  r02a added ~10 of those counters per read with RED.ADD from lane 0, plus one RED.MAX on the launch's "widest
// alignment": a million reads x 11 atomics on one 128-byte line serialise in that L2 slice's atomic unit and back up the SMs'
// memory pipes behind them (long-scoreboard stalls on plain loads, issue slots mostly idle).  Now: registers, flushed when the warp
// moves to another reference (direct-mapped on r mod NA) and at kernel end.
static_assert(C2B_NSCAL <= 32, "one lane per scalar slot");
template <int NA> struct ScAcc { long long v[NA]; int ref[NA]; unsigned wmax; };

template <int NA>
C2B_DEV void sc_init(ScAcc<NA> &A)
{
#pragma unroll
    for (int x = 0; x < NA; x++) { A.v[x] = 0; A.ref[x] = -1; }
    A.wmax = 0;
}

// all lanes call with warp-uniform arguments
template <int NA>
C2B_DEV void sc_acc(ScAcc<NA> &A, const KParams &P, int r, int slot, long long val)
{
    const int lane = wp::lane();
    const int k = NA == 1 ? 0 : (r & (NA - 1));
#pragma unroll
    for (int x = 0; x < NA; x++) {
        if (x != k) continue;
        if (A.ref[x] != r) {
            if (A.ref[x] >= 0 && A.v[x] != 0 && lane < C2B_NSCAL) wp::addg(P.refs[A.ref[x]].scal + lane, A.v[x]);
            A.v[x] = 0; A.ref[x] = r;
        }
        if (lane == slot) A.v[x] += val;
    }
}

template <int NA>
C2B_DEV void sc_flush(ScAcc<NA> &A, const KParams &P)
{
    const int lane = wp::lane();
#pragma unroll
    for (int x = 0; x < NA; x++) {
        if (A.ref[x] >= 0 && A.v[x] != 0 && lane < C2B_NSCAL) wp::addg(P.refs[A.ref[x]].scal + lane, A.v[x]);
        A.v[x] = 0; A.ref[x] = -1;
    }
    if (lane == 0 && A.wmax) wp::maxg(&P.wb->launch.widest, (unsigned long long)A.wmax);      // widest alignment of the launch
    A.wmax = 0;
}

// edited_update (c2b_core.cuh) for the CLASSIFY kernel: what only edited reads add -- size Counters straight to the count
// block (spread addresses), class counters through the warp's accumulators.  References with a coding sequence never get here.
template <int NA>
C2B_DEV void edited_update_acc(ScAcc<NA> &A, const KParams &P, const RefDev &R, int r, const RowOut &o, long long w)
{
    const bool ign_s = P.flags & C2B_F_IGNORE_SUBSTITUTIONS, ign_i = P.flags & C2B_F_IGNORE_INSERTIONS,
               ign_d = P.flags & C2B_F_IGNORE_DELETIONS;
    const bool has_d = !ign_d && o.del_n > 0, has_i = !ign_i && o.ins_n > 0, has_s = !ign_s && o.sub_n > 0;
    if (wp::lane() == 0) {
        unsigned long long *H = R.hist;
        const int hs = P.hstride;
        if (has_i) wp::addg(H + (int64_t)C2B_H_INS_N * hs + o.ins_n, w);
        if (has_d) wp::addg(H + (int64_t)C2B_H_DEL_N * hs + o.del_n, w);
        if (has_s) wp::addg(H + (int64_t)C2B_H_SUB_N * hs + o.sub_n, w);
        const int eff = R.I + (has_i ? o.ins_n : 0) - (has_d ? o.del_n : 0);
        if (eff != R.I) wp::addg(H + (int64_t)C2B_H_EFF_LEN * hs + eff, w);
    }
    if (has_i) sc_acc(A, P, r, C2B_S_INS, w);
    if (has_d) sc_acc(A, P, r, C2B_S_DEL, w);
    if (has_s) sc_acc(A, P, r, C2B_S_SUB, w);
    const int combo = (has_i ? 4 : 0) | (has_d ? 2 : 0) | (has_s ? 1 : 0);
    const int slot = combo == 1 ? C2B_S_ONLY_SUB : combo == 2 ? C2B_S_ONLY_DEL : combo == 3 ? C2B_S_DEL_SUB : combo == 4 ? C2B_S_ONLY_INS
                   : combo == 5 ? C2B_S_INS_SUB : combo == 6 ? C2B_S_INS_DEL : combo == 7 ? C2B_S_INS_DEL_SUB : -1;
    if (slot >= 0) sc_acc(A, P, r, slot, w);
}
struct BSmem {                                         // CLASSIFY kernel, per warp
    uint64_t ops[RG_MAX_REFS][32];                     // op streams of the candidate references
    uint8_t rd[B_RD_BYTES];                            // bytes [off & ~15, ...) of the read buffer
};
struct ColCtx {
    const uint64_t *ops;           // op stream of this slot (shared memory)
    const uint8_t *rd;             // the read's first byte (shared memory)
    int n, J, strand;
    uint32_t mmis, mI, mJ;         // lane m: ballots of step m (mismatching M columns, I columns, J columns) -- filled by colscan0
};
struct ColDec { int op, i, j; uint32_t rdc, rfc, bI, bJ; bool valid; };

C2B_DEV ColDec col_decode(const KParams &P, const RefDev &R, const ColCtx &c, int m, int i0, int j0)
{
    const int lane = wp::lane();
    const uint32_t lt = (1u << lane) - 1u;
    ColDec d;
    const int col = 32 * m + lane;
    d.valid = col < c.n;
    const int q = c.n - 1 - col;
    d.op = OP_NONE;
    if (d.valid) d.op = (int)((c.ops[q >> 5] >> (2 * (q & 31))) & 3ull);
    d.bI = wp::ballot(d.op == OP_I); d.bJ = wp::ballot(d.op == OP_J);
    d.i = i0 + lane - wp::popc(d.bI & lt);
    d.j = j0 + lane - wp::popc(d.bJ & lt);
    d.rdc = '-'; d.rfc = '-';
    if (d.valid && d.op != OP_J) {
        uint32_t ch = c.rd[c.strand ? c.J - 1 - d.j : d.j];
        if (c.strand) ch = P.alpha[P.comp[P.lut[ch]]];
        d.rdc = ch;
    }
    if (d.valid && d.op != OP_I) d.rfc = R.asc[d.i];
    return d;
}

// Pass 0: the two aligned strings (right-aligned in their W-byte slots), matchCount, irregular ends, and the per-step ballots
// pass 1 uses to skip steps in which the read equals the reference.
C2B_DEV ColOut colscan0(const KParams &P, const RefDev &R, ColCtx &c, uint8_t *o_read, uint8_t *o_ref)
{
    const int lane = wp::lane();
    int i0 = 0, j0 = 0, match = 0;
    uint32_t irr = 0;
    c.mmis = c.mI = c.mJ = 0;
    const int nsteps = (c.n + 31) >> 5;
    uint8_t *pr = o_read ? o_read + P.W - c.n + lane : nullptr;
    uint8_t *pf = o_ref ? o_ref + P.W - c.n + lane : nullptr;
#pragma unroll 1
    for (int m = 0; m < nsteps; m++) {
        const ColDec d = col_decode(P, R, c, m, i0, j0);
        const bool eq = d.valid && d.op == OP_M && d.rdc == d.rfc;
        const uint32_t Beq = wp::ballot(eq), Bmis = wp::ballot(d.valid && d.op == OP_M && d.rdc != d.rfc);
        match += wp::popc(Beq);
        const int col = 32 * m + lane;
        irr |= wp::ballot(d.valid && (col == 0 || col == c.n - 1) && !eq);
        if (pr && d.valid) { pr[32 * m] = (uint8_t)d.rdc; pf[32 * m] = (uint8_t)d.rfc; }
        if (lane == m) { c.mmis = Bmis; c.mI = d.bI; c.mJ = d.bJ; }
        const int nv = c.n - 32 * m < 32 ? c.n - 32 * m : 32;
        i0 += nv - wp::popc(d.bI); j0 += nv - wp::popc(d.bJ);
    }
    ColOut o; o.n_match = match; o.irregular = irr != 0;
    return o;
}

// Pass 1: find_indels_substitutions + the per-read quantification, same mode bits and outputs as rows_run (c2b_core.cuh),
// evaluated over alignment columns.  Insertion / deletion runs are closed in the step that holds their first column to the
// right (state carried across steps); flank positions shared by two insertions count once (numpy's fancy-index +=).
// LEGACY = --use_legacy_insertion_quantification as a template parameter: one more flag test inside the scan cost the default
// instantiation registers it does not have (80 at six CTAs per SM): more spills and a slower kernel.
template <bool LEGACY>
C2B_DEVNOINL void colscan1_t(const KParams &P, const RefDev &R, const ColCtx &c, RowOut &o, c2b_edit *ed, long long w, int mode,
                             unsigned long long *Vt = nullptr)
{
    const int lane = wp::lane();
    const uint32_t lt = (1u << lane) - 1u;
    const bool ign_s = P.flags & C2B_F_IGNORE_SUBSTITUTIONS, ign_i = P.flags & C2B_F_IGNORE_INSERTIONS,
               ign_d = P.flags & C2B_F_IGNORE_DELETIONS;
    const bool scal = mode & RM_SCAL, vec = mode & RM_VEC, lenv = mode & RM_LEN, ref1 = mode & RM_REF1;
    unsigned long long *V = ref1 ? Vt : R.vec;
    const int vs = P.vstride, I = R.I;
    int i0 = 0, j0 = 0;
    int del_a = -1;                  // start of the deletion run that is open at the step boundary (-1: none)
    int ins_len = 0;                 // length so far of the insertion run that is open at the step boundary
    int flank_all = -1, flank_win = -1;      // right flank of the last insertion counted in ALL_INS / INS
    const int nsteps = (c.n + 31) >> 5;

    // --use_legacy_insertion_quantification: same rules as rows_run (c2b_core.cuh), COREResources.pyx:190-315
    constexpr bool legacy = LEGACY;
    auto del_run = [&](int a0, int b0) {                   // one deletion run [a0,b0)  (COREResources.pyx:143-160)
        const int size = b0 - a0;
        const int a = (legacy && a0 <= 1) ? 0 : a0, b = (legacy && b0 == I) ? I - 1 : b0;
        const int npos = b > a ? b - a : 0;
        const bool hit = npos > 0 && (int)R.cum[b] - (int)R.cum[a] > 0;
        if (scal) {
            o.n_del_all++; o.n_del_pos += npos;
            if (hit) { o.n_del_win++; o.del_n += size; }
            if (lane == 0 && o.nent < P.edit_cap && ed) {
                c2b_edit e; e.a = (uint16_t)a; e.b = (uint16_t)b; e.type = 3; e.in_window = hit; e.pad = 0;
                e.base = legacy ? (uint8_t)(size - (b - a) + 2) : 0;
                ed[o.nent] = e;
            }
            o.nent++;
        }
        if (legacy && (vec || ref1))
            for (int p = a + lane; p < b; p += 32) wp::addg(V + (int64_t)(ref1 ? C2B_V_R1_ALL_DEL : C2B_V_ALL_DEL) * vs + p, w);
        if (hit && ((vec && !ign_d) || lenv)) {
            for (int p = a + lane; p < b; p += 32) {
                if (vec && !ign_d) wp::addg(V + (int64_t)C2B_V_DEL * vs + p, w);
                if (lenv) wp::addg(V + (int64_t)C2B_V_DEL_LEN * vs + p, w * size);
            }
        }
    };
    auto ins_run = [&](int p1, int size) {                 // insertion of `size` bases between reference positions p1-1 and p1
        if (p1 < 1 || p1 > I - 1) return;                  // before the first / after the last reference base: not an insertion (:117)
        const int p = p1 - 1;
        const bool win = legacy ? (((R.incl[p] | R.incl[p1]) & 1u) != 0) : ((R.incl[p] & 1u) && (R.incl[p1] & 1u));   // both flanks in the window (:120); legacy: either (:284)
        if (scal) {
            o.n_ins_all++;
            if (win) { o.n_ins_win++; o.ins_n += size; }
            if (lane == 0 && o.nent < P.edit_cap && ed) {
                c2b_edit e; e.a = (uint16_t)p; e.b = (uint16_t)size; e.type = 2; e.in_window = win; e.base = 0; e.pad = 0;
                ed[o.nent] = e;
            }
            o.nent++;
        }
        if (lane == 0) {
            if (vec) {
                wp::addg(V + (int64_t)C2B_V_ALL_INS_LEFT * vs + p, w);
                if (p != flank_all) wp::addg(V + (int64_t)C2B_V_ALL_INS * vs + p, w);
                wp::addg(V + (int64_t)C2B_V_ALL_INS * vs + p1, w);
                if (win && !ign_i) {
                    if (p != flank_win) wp::addg(V + (int64_t)C2B_V_INS * vs + p, w);
                    wp::addg(V + (int64_t)C2B_V_INS * vs + p1, w);
                }
            }
            if (ref1) {
                wp::addg(V + (int64_t)C2B_V_R1_ALL_INS_LEFT * vs + p, w);
                if (p != flank_all) wp::addg(V + (int64_t)C2B_V_R1_ALL_INS * vs + p, w);
                wp::addg(V + (int64_t)C2B_V_R1_ALL_INS * vs + p1, w);
            }
            if (lenv && win) {
                wp::addg(V + (int64_t)C2B_V_INS_LEN * vs + p, w * size);
                wp::addg(V + (int64_t)C2B_V_INS_LEN * vs + p1, w * size);
            }
        }
        flank_all = p1;
        if (win) flank_win = p1;
    };

#pragma unroll 1
    for (int m = 0; m < nsteps; m++) {
        const int nv = c.n - 32 * m < 32 ? c.n - 32 * m : 32;
        const uint32_t any = wp::shflu(c.mmis | c.mI | c.mJ, m);
        if (!any && del_a < 0 && ins_len == 0) { i0 += nv; j0 += nv; continue; }      // the read equals the reference here
        const ColDec d = col_decode(P, R, c, m, i0, j0);
        const int p = d.i;
        const bool isM = d.valid && d.op == OP_M, isdel = d.valid && d.op == OP_J;
        const bool differs = isM && d.rdc != d.rfc;
        const bool issub = differs && d.rdc != 'N';                                  // COREResources.pyx:111
        const bool inc_p = (isM || isdel) && (R.incl[p] & 1u);
        int rcode = 0;
        if (differs) rcode = P.lut[d.rdc];
        if (scal) {
            const uint32_t Bs = wp::ballot(issub), Bsw = wp::ballot(issub && inc_p);
            o.n_sub_all += wp::popc(Bs); o.sub_n += wp::popc(Bsw);
            if (Bs) {
                const int idx = o.nent + wp::popc(Bs & lt);
                if (issub && idx < P.edit_cap && ed) {
                    c2b_edit e; e.a = (uint16_t)p; e.b = 0; e.type = 1; e.in_window = inc_p; e.base = (uint8_t)d.rdc; e.pad = 0;
                    ed[idx] = e;
                }
                o.nent += wp::popc(Bs);
            }
        }
        if (vec) {
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
            if (isdel && !legacy) wp::addg(V + (int64_t)C2B_V_R1_ALL_DEL * vs + p, w);
            if (issub) wp::addg(V + (int64_t)C2B_V_R1_ALL_SUB * vs + p, w);
            if (isdel || differs) {
                const int rc = R.rcode[p];
                wp::addg(V + (int64_t)(C2B_V_R1_BASEDEV0 + (isdel ? P.nq : rcode)) * vs + p, w);
                if (rc != 255) wp::addg(V + (int64_t)(C2B_V_R1_BASEDEV0 + rc) * vs + p, -w);
            }
        }
        // runs: a set bit of E* marks the first column to the right of a run (the column past the alignment closes a
        // run that reaches its end); ref index of lane x of this step = i0 + x - popc(bI below x)
        const uint32_t vmask = nv == 32 ? 0xffffffffu : ((1u << nv) - 1u);
        auto ref_at = [&](int x) { return i0 + x - wp::popc(d.bI & ((1u << x) - 1u)); };
        uint32_t events;
        {
            const uint32_t D = d.bJ, Dsh = (D << 1) | (del_a >= 0 ? 1u : 0u);
            const uint32_t Ds = D & ~Dsh, De = ~D & Dsh;                 // starts / first column after a run
            const uint32_t Iw = d.bI, Ish = (Iw << 1) | (ins_len > 0 ? 1u : 0u);
            const uint32_t Is = Iw & ~Ish, Ie = ~Iw & Ish;
            events = De | Ie;
            // close runs in column order (deletion and insertion runs never touch, Align.pyx:394-413)
            uint32_t rem = events;
            // a run that ends exactly at the alignment's end inside this step closes at column nv (bit nv, if nv < 32)
            while (rem) {
                const int eb = wp::ffs(rem) - 1;
                rem &= rem - 1;
                if ((De >> eb) & 1u) {
                    const uint32_t below = Ds & ((1u << eb) - 1u);
                    const int a = below ? ref_at(31 - wp::clz(below)) : del_a;
                    del_run(a, ref_at(eb));
                    del_a = -1;
                } else {
                    const uint32_t below = Is & ((1u << eb) - 1u);
                    const int sb = below ? 31 - wp::clz(below) : -1;
                    const int size = sb >= 0 ? eb - sb : ins_len + eb;
                    ins_run(ref_at(eb), size);
                    ins_len = 0;
                }
            }
            // runs still open at the end of the step
            if ((D >> 31) & 1u) { if (del_a < 0) { const uint32_t s = Ds; del_a = ref_at(31 - wp::clz(s)); } }
            if ((Iw >> 31) & 1u) {
                const uint32_t s = Is;
                if (ins_len > 0 && !s) ins_len += 32;                                  // the whole step is one run
                else ins_len = 32 - (31 - wp::clz(s));
            }
            (void)vmask;
        }
        i0 += nv - wp::popc(d.bI); j0 += nv - wp::popc(d.bJ);
    }
    if (del_a >= 0) del_run(del_a, I);                     // a deletion that reaches the end of the alignment
    // an insertion run that reaches the end of the alignment lies after the last reference base: not counted
}

C2B_DEV void colscan1(const KParams &P, const RefDev &R, const ColCtx &c, RowOut &o, c2b_edit *ed, long long w, int mode,
                      unsigned long long *Vt = nullptr)
{
    if (P.flags & C2B_F_LEGACY_INS) colscan1_t<true>(P, R, c, o, ed, w, mode, Vt);
    else colscan1_t<false>(P, R, c, o, ed, w, mode, Vt);
}

// Classification + counts of one read whose alignments to references r_begin..r_end-1 were produced by the ALIGN kernel:
// the body of finish_read (c2b_core.cuh) over column scans instead of the shared-memory row view.
// The kernel loop loads a read's inputs in two stages, each issued a full iteration before its values are used, so that no
// load's latency is waited for: stage A (two reads ahead) the per-read scalars -- offsets, first meta word, count, weight,
// reference id; stage B (one read ahead, addresses from A) the op streams and the read's bytes.
struct BPreA { int64_t off; int J, r_begin; uint32_t gm0; int cnt, qw; };
struct BPre { uint64_t ops[RG_MAX_REFS]; uint4 bytes; uint32_t gm[RG_MAX_REFS]; int64_t off; int J, r_begin, nref, cnt, qw; bool go; };

C2B_DEV BPreA classify_pre_a(const KParams &P, int64_t rd)
{
    BPreA a;
    a.r_begin = P.ref_id ? P.ref_id[rd] : 0;
    a.off = P.offsets[rd];
    a.J = (int)(P.offsets[rd + 1] - a.off);
    a.gm0 = wp::ldcg(P.gmeta + rd * P.out_refs);                        // = oslot(P, rd, r_begin)
    a.cnt = P.count ? P.count[rd] : 1;
    a.qw = P.qweight ? P.qweight[rd] : a.cnt;
    return a;
}

template <bool ONE>
C2B_DEV BPre classify_pre_b(const KParams &P, int64_t rd, const BPreA &a, int64_t total_bytes)
{
    const int lane = wp::lane();
    BPre b;
    b.r_begin = a.r_begin;
    b.nref = (ONE || P.ref_id) ? 1 : P.n_refs;
    const int64_t slot0 = rd * P.out_refs;
    b.go = (a.gm0 >> 24) == GM_ALIGNED;                                  // aligned by the ALIGN kernel (all candidates or none)
    b.off = a.off; b.J = a.J; b.cnt = a.cnt; b.qw = a.qw;
    b.bytes = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int k = 0; k < (ONE ? 1 : RG_MAX_REFS); k++) { b.ops[k] = ~0ull; b.gm[k] = 0; }
    if (!b.go) return b;
    b.gm[0] = a.gm0;
#pragma unroll
    for (int k = 0; k < (ONE ? 1 : RG_MAX_REFS); k++) {
        if (k < b.nref) {
            if (k > 0) b.gm[k] = wp::ldcg(P.gmeta + slot0 + k);
            if (lane < P.NW) b.ops[k] = wp::ldcg64(P.gops + (slot0 + k) * P.NW + lane);
        }
    }
    // 16-byte windows from the aligned address at or below the read's first byte (alignment of the ABSOLUTE address)
    const uint8_t *p0 = P.reads + b.off;
    const uint8_t *wa = p0 - ((uintptr_t)p0 & 15) + 16 * lane;
    if (wa < p0 + b.J) {
        if (wa >= P.reads && wa + 16 <= P.reads + total_bytes) b.bytes = wp::ldg4u(reinterpret_cast<const uint4 *>(wa));
        else {                                               // first / last bytes of the buffer: no load outside it
            uint32_t w[4] = {0, 0, 0, 0};
            for (int x = 0; x < 16; x++) if (wa + x >= P.reads && wa + x < P.reads + total_bytes) w[x >> 2] |= (uint32_t)wa[x] << (8 * (x & 3));
            b.bytes = make_uint4(w[0], w[1], w[2], w[3]);
        }
    }
    return b;
}

template <bool ONE>
C2B_DEV void classify_stage(const BPre &b, BSmem &S)
{
    const int lane = wp::lane();
#pragma unroll
    for (int k = 0; k < (ONE ? 1 : RG_MAX_REFS); k++) if (k < b.nref) S.ops[k][lane] = b.ops[k];
    reinterpret_cast<uint4 *>(S.rd)[lane] = b.bytes;
}

// Pass 0's result for reference r (alignment of n columns on `strand`) -> the alignment record and the best-reference bookkeeping
template <int NA>
C2B_DEV void note_aln(c2b_read_rec &rec, c2b_aln_rec &a, const RefDev &R, int r, const ColOut &co, int n, int strand, ScAcc<NA> &A)
{
    init_aln(a, 0);
    a.n_match = (uint16_t)co.n_match; a.aln_len = (uint16_t)n; a.strand = (uint8_t)strand;
    a.score_milli = score_milli(co.n_match, n);
    a.irregular_ends = (uint8_t)co.irregular;
    note_score(rec, R, r, a.score_milli);
    if ((unsigned)n > A.wmax) A.wmax = (unsigned)n;               // widest alignment of the launch
}

// The per-winner part of classify_read: reference r's alignment, a winner of read rd -> its alignment record, edit list,
// count vectors and scalars.  scan(o, ed, mode) runs the alignment's column scan with colscan1's mode bits (RM_SCAL, RM_VEC,
// RM_LEN); `a` is the record note_aln filled (used when the read has one candidate reference: multi reloads it).
template <bool ONE, class Scan>
C2B_DEV void classify_winner(const KParams &P, const RefDev &R, int64_t rd, int r, c2b_read_rec &rec, const c2b_aln_rec &a,
                             bool multi, bool ambiguous, int nth, long long cnt, long long w, ScAcc<ONE ? 1 : RG_MAX_REFS> &A,
                             const Scan &scan)
{
    const int lane = wp::lane();
    const bool expand = P.flags & C2B_F_EXPAND_AMBIGUOUS, first = P.flags & C2B_F_ASSIGN_FIRST;
    const bool ign_s = P.flags & C2B_F_IGNORE_SUBSTITUTIONS, ign_i = P.flags & C2B_F_IGNORE_INSERTIONS,
               ign_d = P.flags & C2B_F_IGNORE_DELETIONS;
    const bool two_scans = (P.flags & C2B_F_DISCARD_INDEL_READS) != 0;
    rec.best_ref = (int16_t)r;                          // best_match_name = last winner (:768)
    RowOut o; o.ins_n = o.del_n = o.sub_n = 0; o.n_ins_all = o.n_ins_win = o.n_del_all = o.n_del_win = 0;
    o.n_del_pos = o.n_sub_all = 0; o.nent = 0;
    c2b_edit *ed = P.edits ? P.edits + oslot(P, rd, r) * (int64_t)P.edit_cap : nullptr;
    const bool counted = !ambiguous && (!first || nth == 0) && w > 0;
    // with no ignore_* flag a window indel makes the read MODIFIED, so the length vectors (:4104-4115) can be updated in
    // the same scan; otherwise (and under --discard_indel_reads) the scalars decide first
    const bool len_inline = counted && !two_scans && !ign_i && !ign_d;
    scan(o, ed, RM_SCAL | ((counted && !two_scans) ? RM_VEC : 0) | (len_inline ? RM_LEN : 0));
    const bool has_d = !ign_d && o.del_n > 0, has_i = !ign_i && o.ins_n > 0, has_s = !ign_s && o.sub_n > 0;
    const bool modified = has_d || has_i || has_s;     // CRISPRessoCORE.py:746-753 (same truth table)
    uint32_t astatus = 0;
    if (P.edits && o.nent > P.edit_cap) astatus |= C2B_ST_EDIT_OVERFLOW;
    if (counted) {
        const bool discard = two_scans && (o.del_n > 0 || o.ins_n > 0);
        if (discard) sc_acc(A, P, r, C2B_S_DISCARDED, w);
        else {
            const bool entered = modified || R.tem != 0;
            const bool lenv = !len_inline && entered && (o.n_ins_win > 0 || o.n_del_win > 0);
            if (two_scans || lenv) scan(o, nullptr, (two_scans ? RM_VEC : 0) | (lenv ? RM_LEN : 0));
            if (entered) edited_update_acc(A, P, R, r, o, w);              // references with a coding sequence never get here
            sc_acc(A, P, r, C2B_S_TOTAL, w);
            sc_acc(A, P, r, modified ? C2B_S_MODIFIED : C2B_S_UNMODIFIED, w);
        }
    } else if (ambiguous && nth == 0 && w > 0) sc_acc(A, P, r, C2B_S_AMBIGUOUS_W, w);
    if (counted && (two_scans || expand)) {
        const bool discarded = two_scans && (o.del_n > 0 || o.ins_n > 0), joined = !ONE && expand && !first && rec.n_winners > 1;   // assign-first is tested first (:780-785)
        if (discarded != joined) sc_acc(A, P, r, modified ? C2B_S_CLASS_MODIFIED : C2B_S_CLASS_UNMODIFIED, discarded ? w : -w);
    }
    int irr = 0;
    if (lane == 0) {
        c2b_aln_rec b = multi ? load_aln(P.alns + oslot(P, rd, r)) : a;
        b.insertion_n = (uint16_t)o.ins_n; b.deletion_n = (uint16_t)o.del_n; b.substitution_n = (uint16_t)o.sub_n;
        b.n_ins_all = (uint16_t)o.n_ins_all; b.n_ins_win = (uint16_t)o.n_ins_win;
        b.n_del_all = (uint16_t)o.n_del_all; b.n_del_win = (uint16_t)o.n_del_win;
        b.n_del_pos_all = (uint16_t)o.n_del_pos; b.n_sub_all = (uint16_t)o.n_sub_all;
        b.n_edits = (uint16_t)o.nent; b.modified = modified; b.status |= (uint8_t)astatus;
        irr = b.irregular_ends;
        P.alns[oslot(P, rd, r)] = b;
    }
    irr = wp::shfl(irr, 0);
    rec.status |= astatus;
    // aln_stats of the serial process_fastq branch use best_match_name only (:1971-1979): the LAST winner
    const bool is_last = (rec.winner_mask >> (r & 31)) >> 1 == 0;
    if (is_last) {
        const long long total_mods = o.n_ins_all + o.n_del_pos + o.n_sub_all;
        const long long in_win = o.sub_n + o.del_n + o.ins_n;
        sc_acc(A, P, r, C2B_S_N_GLOBAL_SUBS, cnt * o.n_sub_all);
        sc_acc(A, P, r, C2B_S_N_SUBS_OUTSIDE_WINDOW, cnt * (o.n_sub_all - o.sub_n));
        sc_acc(A, P, r, C2B_S_N_MODS_IN_WINDOW, cnt * in_win);
        sc_acc(A, P, r, C2B_S_N_MODS_OUTSIDE_WINDOW, cnt * (total_mods - in_win));
        if (irr) sc_acc(A, P, r, C2B_S_N_READS_IRREGULAR_ENDS, cnt);
        sc_acc(A, P, r, C2B_S_N_ALIGNED_UNIQUE, 1);
        sc_acc(A, P, r, C2B_S_N_ALIGNED_COUNT, cnt);
    }
}

template <bool ONE>
C2B_DEV void classify_read(const KParams &P, int64_t rd, const BPre &pre, const BSmem &S, ScAcc<ONE ? 1 : RG_MAX_REFS> &A)
{
    const int lane = wp::lane();
    const int r_begin = pre.r_begin;
    const int r_end = r_begin + pre.nref;
    const int64_t off = pre.off;
    const int J = pre.J;
    const bool multi = !ONE && (r_end - r_begin) > 1;

    c2b_read_rec rec; rec.winner_mask = 0; rec.best_score_milli = -1000; rec.best_ref = -1; rec.n_winners = 0;
    rec.ambiguous = 0; rec.status = 0;
    ColCtx cx[ONE ? 1 : RG_MAX_REFS];
    c2b_aln_rec a; init_aln(a, 0);
#pragma unroll 1
    for (int r = r_begin; r < r_end; r++) {
        const RefDev &R = refdev(P, r);
        const int64_t slot = oslot(P, rd, r);
        ColCtx &c = cx[ONE ? 0 : r - r_begin];
        const uint32_t gm = pre.gm[ONE ? 0 : r - r_begin];
        c.ops = S.ops[ONE ? 0 : r - r_begin]; c.rd = S.rd + (int)((uintptr_t)(P.reads + off) & 15); c.n = (int)(gm & 0xffffu); c.J = J; c.strand = (int)((gm >> 16) & 1u);
        uint8_t *o_read = P.strings ? P.strings + (slot * 2) * (int64_t)P.W : nullptr;
        const ColOut co = colscan0(P, R, c, o_read, o_read ? o_read + P.W : nullptr);
        note_aln(rec, a, R, r, co, c.n, c.strand, A);
        if (lane == 0 && multi) P.alns[slot] = a;
    }
    if (multi) wp::sync();
    if (rec.best_score_milli <= 0) {
        rec.winner_mask = 0; rec.n_winners = 0;
        if (lane == 0) { if (!multi) P.alns[oslot(P, rd, r_begin)] = a; P.recs[rd] = rec; }
        return;
    }
    const bool expand = P.flags & C2B_F_EXPAND_AMBIGUOUS, first = P.flags & C2B_F_ASSIGN_FIRST;
    const bool ambiguous = !ONE && rec.n_winners > 1 && !first && !expand;     // CRISPRessoCORE.py:780-785
    rec.ambiguous = ambiguous;
    const long long w = pre.qw;
    int nth = 0;
#pragma unroll 1
    for (int r = r_begin; r < r_end; r++) {
        if (!((rec.winner_mask >> (r & 31)) & 1u)) continue;
        const RefDev &R = refdev(P, r);
        const ColCtx &c = cx[ONE ? 0 : r - r_begin];
        classify_winner<ONE>(P, R, rd, r, rec, a, multi, ambiguous, nth, pre.cnt, w, A,
                             [&](RowOut &o, c2b_edit *ed, int mode) { colscan1(P, R, c, o, ed, w, mode); });
        nth++;
    }
    // HDR / prime editing: reads assigned to another reference are also classified on their alignment to reference 0
    if (!ONE && (P.flags & C2B_F_HDR_REF1) && multi && r_begin == 0 && !ambiguous && w > 0) {
        const uint32_t eff = first ? (rec.winner_mask & (0u - rec.winner_mask)) : rec.winner_mask;   // aln_ref_names
        if (eff != 1u) {                                    // not "aligned to reference 0 only" (:4234)
            const RefDev &R0 = P.refs[0];
            RowOut dummy; dummy.ins_n = dummy.del_n = dummy.sub_n = 0; dummy.n_ins_all = dummy.n_ins_win = 0;
            dummy.n_del_all = dummy.n_del_win = dummy.n_del_pos = dummy.n_sub_all = 0; dummy.nent = 0;
            for (int r = 1; r < r_end; r++) {
                if (!((eff >> (r & 31)) & 1u)) continue;
                colscan1(P, R0, cx[0], dummy, nullptr, w, RM_REF1, P.refs[r].vec);
                sc_acc(A, P, r, C2B_S_REF1_W, w);
            }
        }
    }
    if (lane == 0) P.recs[rd] = rec;
}

// The CLASSIFY kernel's loop for warp `warp` of `nwarps`: one aligned read per warp, reads strided over the warps -- every
// read, or (after the diagonal tier, which classifies the reads it proves) the entries of its list: P.pair_order, *P.n_dev.
template <bool ONE>
C2B_DEV void classify_loop(const KParams &P, BSmem &S, int64_t warp, int64_t nwarps)
{
    const int64_t nw = nwarps;
    const int64_t total_bytes = P.offsets[P.n_reads];
    const int64_t n = nreads(P);
    int64_t x = warp;                                                    // position in the read order
    if (x >= n) return;
    ScAcc<ONE ? 1 : RG_MAX_REFS> acc;
    sc_init(acc);
    // two-deep input pipeline: stage A of position x + 2 nw and stage B of x + nw are in flight while x is classified; the
    // read at x + 3 nw is looked up one iteration before its stage A needs it (a list entry, then its offsets: two round trips)
    int32_t rd = (int32_t)read_at(P, x), rd1 = 0, rd2 = 0;
    BPreA a1 = classify_pre_a(P, rd);
    BPre pre = classify_pre_b<ONE>(P, rd, a1, total_bytes);
    if (x + nw < n) { rd1 = (int32_t)read_at(P, x + nw); a1 = classify_pre_a(P, rd1); }
    if (x + 2 * nw < n) rd2 = (int32_t)read_at(P, x + 2 * nw);
    while (x < n) {
        const BPre cur = pre;
        const int32_t rc = rd;
        if (cur.go) classify_stage<ONE>(cur, S);
        wp::sync();
        const int64_t nxt = x + nw;
        if (nxt < n) {
            pre = classify_pre_b<ONE>(P, rd1, a1, total_bytes);
            rd = rd1;
            if (nxt + nw < n) { a1 = classify_pre_a(P, rd2); rd1 = rd2; }
            if (nxt + 2 * nw < n) rd2 = (int32_t)read_at(P, nxt + 2 * nw);
        }
        if (cur.go) classify_read<ONE>(P, rc, cur, S, acc);
        wp::sync();
        x = nxt;
    }
    sc_flush(acc, P);
}

// ---------------------------------------------------------------------------------------- diagonal tier (tier 0)
// A read as long as its amplicon whose ungapped score on the main diagonal beats every other path is aligned there, with no
// DP: it scores strictly above RefDev::dg_thr4 (the bound on paths with an interior gap run, on offset diagonals past dg_S and
// on paths through the reference's min_score borders) and strictly above the exact score of each offset diagonal 1..dg_S with
// its two edge runs.  Then the diagonal is the unique optimum and the reference's traceback returns it (DESIGN.md section 3).
// The tier also classifies the reads it proves (diag_classify), so the narrow tier and CLASSIFY only see the others.
// One read per warp, 32 consecutive reads per unit; the unit's unproved reads go, in order and with one atomic, on the tier-0
// list (P.left0) that CLASSIFY works through.  With routing (P.route) each of them also goes either on the narrow tier's list
// (P.left1) or straight onto the tier-2 list (P.left2) that the wide ring works through (route_read).
constexpr int DG_PROVED = 0, DG_KEEP = 1, DG_ROUTE = 2;     // diag_read: proved / for the narrow tier / for the wide ring
struct DSmem {                                         // diagonal tier, per warp
    uint4 pl[2][10];                                   // the read's and the reference's codes as bit planes, 32 columns per word
    uint8_t raw[2][RG_COMBO + 32];                     // the bytes of the unit's next reads, from the 16-byte line at or below each (diag_stage)
    int32_t pl_ref;                                    // reference whose planes are in pl[1] (-1: none)
    uint8_t fw[RG_COMBO], rc[RG_COMBO];
    uint8_t lut[256];
    int64_t off[33];
    int64_t total_bytes;                               // of the read buffer
    int32_t ref[32], cnt[32], qw[32];
    int32_t npop;                                      // reads this warp scored by popcounts
};

// Bit planes of alphabet codes, 32 columns per word (x: code bit 0, y: code bit 1, z: code in 0..3): the columns where two
// words hold the same code in 0..3; columns x + t of the word pair (lo, hi), 0 <= t < 32; the columns below n of a word
C2B_DEV uint32_t pl_match(uint4 a, uint4 b) { return ~((a.x ^ b.x) | (a.y ^ b.y)) & a.z & b.z; }
C2B_DEV uint4 pl_shifted(uint4 lo, uint4 hi, int t)
{
    return make_uint4(wp::funnel_r(lo.x, hi.x, t), wp::funnel_r(lo.y, hi.y, t), wp::funnel_r(lo.z, hi.z, t), 0u);
}
C2B_DEV uint32_t pl_below(int n) { return n >= 32 ? ~0u : n <= 0 ? 0u : (1u << n) - 1u; }

// classify_read<true> for a read the tier proved: I columns of OP_M on the main diagonal, no gap column.  c: the read as
// alphabet codes in the aligned strand; column p's read character is P.alpha[c[p]], which is how col_decode spells it (the
// lookup table maps exactly the alphabet's characters, and a read with any other symbol is never proved).  planes: the read
// and the amplicon hold codes 0..3 only and S.pl holds their bit planes (diag_read), so a column differs iff its codes do.
C2B_DEV void diag_classify(const KParams &P, const DSmem &S, const RefDev &R, const uint8_t *c, int64_t rd, int r, int strand,
                           long long cnt, long long w, ScAcc<1> &A, bool planes)
{
    const int lane = wp::lane(), I = R.I;
    const uint32_t lt = (1u << lane) - 1u;
    const int64_t slot = oslot(P, rd, r);
    const int nsteps = (I + 31) >> 5;
    // pass 0 (colscan0): the two strings right-aligned in their W-byte slots, matchCount, irregular ends; lane m keeps the
    // ballot of step m's mismatching columns
    uint8_t *o_read = P.strings ? P.strings + (slot * 2) * (int64_t)P.W + P.W - I : nullptr;
    int match = 0;
    uint32_t irr = 0, mmis = 0;
    if (planes) {                                    // the ballots from the planes; the strings' loads overlap
        mmis = lane < nsteps ? ~pl_match(S.pl[0][lane], S.pl[1][lane]) & pl_below(I - 32 * lane) : 0u;
        int k = wp::popc(mmis);
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) k += wp::shfl_xor(k, d);
        match = I - k;
        irr = (wp::shflu(mmis, 0) & 1u) | ((wp::shflu(mmis, nsteps - 1) >> ((I - 1) & 31)) & 1u);
        if (o_read)
#pragma unroll 4
            for (int m = 0; m < nsteps; m++) {
                const int p = 32 * m + lane;
                if (p < I) { o_read[p] = (uint8_t)P.alpha[c[p]]; o_read[P.W + p] = R.asc[p]; }
            }
    } else {
#pragma unroll 1
        for (int m = 0; m < nsteps; m++) {
            const int p = 32 * m + lane;
            const bool valid = p < I;
            const uint32_t rdc = valid ? P.alpha[c[p]] : 0u, rfc = valid ? R.asc[p] : 0u;
            const uint32_t Bmis = wp::ballot(valid && rdc != rfc);
            match += wp::popc(wp::ballot(valid && rdc == rfc));
            irr |= wp::ballot(valid && (p == 0 || p == I - 1) && rdc != rfc);
            if (o_read && valid) { o_read[p] = (uint8_t)rdc; o_read[P.W + p] = (uint8_t)rfc; }
            if (lane == m) mmis = Bmis;
        }
    }
    ColOut co; co.n_match = match; co.irregular = irr != 0;
    c2b_read_rec rec; rec.winner_mask = 0; rec.best_score_milli = -1000; rec.best_ref = -1; rec.n_winners = 0;
    rec.ambiguous = 0; rec.status = 0;
    c2b_aln_rec a;
    note_aln(rec, a, R, r, co, I, strand, A);
    if (rec.best_score_milli <= 0) {
        rec.winner_mask = 0; rec.n_winners = 0;
        if (lane == 0) { P.alns[slot] = a; P.recs[rd] = rec; }
        return;
    }
    // colscan1 without gap columns: every differing column is a substitution unless the read has N there; no runs, no flanks
    auto scan = [&](RowOut &o, c2b_edit *ed, int mode) {
        const bool scal = mode & RM_SCAL, vec = mode & RM_VEC, ign_s = P.flags & C2B_F_IGNORE_SUBSTITUTIONS;
        unsigned long long *V = R.vec;
        const int vs = P.vstride;
#pragma unroll 1
        for (int m = 0; m < nsteps; m++) {
            const uint32_t bm = wp::shflu(mmis, m);
            if (!bm) continue;                                                       // the read equals the reference here
            const int p = 32 * m + lane;
            const bool differs = (bm >> lane) & 1u;
            const uint32_t rdc = differs ? P.alpha[c[p]] : 0u;
            const bool issub = differs && rdc != 'N';                                // COREResources.pyx:111
            const bool inc_p = differs && (R.incl[p] & 1u);
            const int rcode = differs ? S.lut[rdc] : 0;
            if (scal) {
                const uint32_t Bs = wp::ballot(issub), Bsw = wp::ballot(issub && inc_p);
                o.n_sub_all += wp::popc(Bs); o.sub_n += wp::popc(Bsw);
                if (Bs) {
                    const int idx = o.nent + wp::popc(Bs & lt);
                    if (issub && idx < P.edit_cap && ed) {
                        c2b_edit e; e.a = (uint16_t)p; e.b = 0; e.type = 1; e.in_window = inc_p; e.base = (uint8_t)rdc; e.pad = 0;
                        ed[idx] = e;
                    }
                    o.nent += wp::popc(Bs);
                }
            }
            if (vec) {
                if (issub) {
                    wp::addg(V + (int64_t)C2B_V_ALL_SUB * vs + p, w);
                    if (!ign_s) {
                        wp::addg(V + (int64_t)(C2B_V_SUBBASE0 + rcode) * vs + p, w);
                        if (inc_p) wp::addg(V + (int64_t)C2B_V_SUB * vs + p, w);
                    }
                }
                if (differs) {                                   // all_base_count_vectors as deviation from "read == ref"
                    const int rc = R.rcode[p];
                    wp::addg(V + (int64_t)(C2B_V_BASEDEV0 + rcode) * vs + p, w);
                    if (rc != 255) wp::addg(V + (int64_t)(C2B_V_BASEDEV0 + rc) * vs + p, -w);
                }
            }
        }
    };
    classify_winner<true>(P, R, rd, r, rec, a, false, false, 0, cnt, w, A, scan);
    if (lane == 0) P.recs[rd] = rec;
}

// Routing test for an unproved read of the amplicon's length (J == I <= 256, every base in the alphabet, one strand); D: its
// exact score on the main diagonal.  -> DG_KEEP when a path inside the narrow band provably beats that tier's bound (so the
// narrow tier settles the read), DG_ROUTE otherwise.  The paths tried: the main diagonal up to split p >= 1, one interior gap
// run of t = |s| columns, offset diagonal s (read j = reference i + s) to the end, then s's edge run.  Index x counts read
// columns for s < 0 (read x against reference x + t) and reference rows for s > 0 (reference x against read x + t); with m0 /
// ms the match bits of diagonal 0 / s over x, F(p) = (m0 below p) + (ms from p on), and the path scores at least
// rt_mx F(p) + rt_c[s] + its gap run's incentives (a matched column scores at least the least match score, any other column
// at least the least score).  Lane s + 16 takes offset s and finds its best split among the block ends p = 32, 64, ..
// (clamped to I - t); the best lane's 64 splits around its block end are then scanned exactly, incentives included.  A read
// is kept iff that lower bound beats rt_thr; any other read costs the wide ring what the narrow tier would have wasted on it.
// S.pl holds the read's and the amplicon's bit planes (diag_read).
C2B_DEV int route_read(const RefDev &R, const DSmem &S, int D)
{
    if (!R.rt_ok || D > R.rt_thr) return DG_KEEP;            // no bound for this reference / the diagonal alone beats it
    const int lane = wp::lane(), I = R.I, nb = (I + 31) >> 5;
    const int s = lane - 16, t = s < 0 ? -s : s, cs = R.rt_c[lane];
    const uint4 *Ap = S.pl[s < 0 ? 0 : 1], *Bp = S.pl[s < 0 ? 1 : 0];
    int run = 0, best = RT_OFF, bb = 1, mst = 0;             // run: F(32 (b + 1)) - mst; bb: first block end attaining best
#pragma unroll 1
    for (int b = 0; b < nb; b++) {
        const uint32_t m0 = pl_match(S.pl[0][b], S.pl[1][b]) & pl_below(I - t - 32 * b);
        const uint32_t ms = pl_match(Ap[b], pl_shifted(Bp[b], Bp[b + 1], t));
        const int k = wp::popc(ms);
        run += wp::popc(m0) - k; mst += k;
        if (run > best) { best = run; bb = b + 1; }
    }
    const int val = cs == RT_OFF ? RT_OFF : R.rt_mx * (mst + best) + cs;
    int vmax = val;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) { const int o = wp::shfl_xor(vmax, d); if (o > vmax) vmax = o; }
    if (vmax == RT_OFF) return DG_ROUTE;                     // no offset to try: the diagonal alone, which does not beat the bound
    const int L = wp::ffs(wp::ballot(val == vmax)) - 1;
    const int s1 = L - 16, t1 = s1 < 0 ? -s1 : s1, w0 = wp::shfl(bb, L) - 1, F1 = wp::shfl(mst + best, L), c1 = wp::shfl(cs, L);
    const uint4 *A1 = S.pl[s1 < 0 ? 0 : 1], *B1 = S.pl[s1 < 0 ? 1 : 0];
    uint32_t m0w[2], msw[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        m0w[h] = pl_match(S.pl[0][w0 + h], S.pl[1][w0 + h]) & pl_below(I - t1 - 32 * (w0 + h));
        msw[h] = pl_match(A1[w0 + h], pl_shifted(B1[w0 + h], B1[w0 + h + 1], t1));
    }
    // lane l: columns 2l, 2l + 1 of blocks w0, w0 + 1; F at the splits after them from F(32 w0) and a prefix sum over the lanes
    const int F0 = F1 - (wp::popc(m0w[0]) - wp::popc(msw[0]));
    const uint32_t a = lane < 16 ? m0w[0] : m0w[1], bm = lane < 16 ? msw[0] : msw[1];
    const int j = (2 * lane) & 31;
    const int e0 = (int)((a >> j) & 1u) - (int)((bm >> j) & 1u), e1 = (int)((a >> (j + 1)) & 1u) - (int)((bm >> (j + 1)) & 1u);
    int incl = e0 + e1;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int v = wp::shfl_up(incl, d); if (lane >= d) incl += v; }
    const int imul = s1 < 0 ? 1 : t1;                        // a deletion collects its row's incentive once, an insertion per column
    int e = RT_OFF;
    auto cand = [&](int p, int F) {
        if (p >= 1 && p <= I - t1) { const int v = R.rt_mx * F + imul * (R.g4[p] >> 2) + c1; if (v > e) e = v; }
    };
    const int pa = 32 * w0 + 2 * lane + 1;
    cand(pa, F0 + incl - e1);
    cand(pa + 1, F0 + incl);
    if (lane == 0) cand(32 * w0, F0);
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) { const int o = wp::shfl_xor(e, d); if (o > e) e = o; }
    return e > R.rt_thr ? DG_KEEP : DG_ROUTE;
}

// DG_PROVED if read rd is proved (op stream, meta word and classification written), else where it goes next (DG_KEEP: the
// narrow tier, DG_ROUTE: straight to the wide ring; DG_KEEP whenever routing is off); all lanes call with warp-uniform arguments.
// bytes: the read's J bytes (S.raw)
C2B_DEV int diag_read(const KParams &P, DSmem &S, int64_t rd, const uint8_t *bytes, int J, int r, long long cnt, long long w,
                      ScAcc<1> &A)
{
    const int lane = wp::lane();
    const RefDev &R = refdev(P, r);
    const int I = R.I;
    // the reads the narrow tier would take (one candidate reference, packed ring admissible), of the amplicon's length
    if (!R.dg_ok || J != I || J > RG_COMBO || J + 32 > P.TS || J > R.pk_maxJ || I + J > PK_MAX_ALN) return DG_KEEP;
    const bool bad = load_codes_a(P, S.lut, bytes, J, S.fw, S.rc);
    wp::sync();
    // a symbol outside the alphabet or a seed test that wants both strands: the narrow tier only carries such a read to tier 2
    if (bad) return P.route ? DG_ROUTE : DG_KEEP;
    const int mode = strand_mode(P, R, S.fw, J);
    if (mode == 2) return P.route ? DG_ROUTE : DG_KEEP;     // both strands: the DP decides which one
    const uint8_t *c = mode == 1 ? S.rc : S.fw;
    // the read's bit planes in the aligned strand (lane b keeps word b; zero from word nb on) and, once per reference, the
    // amplicon's: the popcount scores and route_read share them.  Either user implies I <= 256: 8 words and 2 zero words.
    const int nb = (I + 31) >> 5, dS = R.dg_S;
    uint4 rp = make_uint4(0u, 0u, 0u, 0u);
    bool acgt = false;                               // every column of the read holds a code in 0..3
    if (R.dg_two || R.rt_ok) {
        for (int b = 0; b < nb; b++) {
            const int x = 32 * b + lane, q = x < I ? c[x] : 255;
            const uint32_t p0 = wp::ballot(q & 1), p1 = wp::ballot(q & 2), v = wp::ballot(q < 4);
            if (lane == b) rp = make_uint4(p0, p1, v, 0u);
        }
        acgt = wp::ballot(lane < nb && rp.z != pl_below(I - 32 * lane)) == 0;
        if (lane < nb + 2) S.pl[0][lane] = rp;
        const bool fresh = S.pl_ref != r;
        wp::sync();
        if (fresh) {
            if (lane < nb + 2) S.pl[1][lane] = R.rt_pl[lane];
            if (lane == 0) S.pl_ref = r;
        }
        wp::sync();
    }
    int D;                                           // 4 x ungapped score on the main diagonal
    bool proved;
    if (R.dg_two && acgt) {
        // every column scores dg_a4 (read code == amplicon code) or dg_b4: the same sums as below, grouped by the match
        // counts of diagonal 0 and of offset s over its I - |s| columns (read base k + s against reference row k)
        if (lane == 0) S.npop++;
        const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
        const uint4 rf = lane < nb ? S.pl[1][lane] : z4, rf1 = lane < nb ? S.pl[1][lane + 1] : z4, rp1 = lane < nb ? S.pl[0][lane + 1] : z4;
        auto total = [](int v) {                     // over lanes 0..7 (the words), to every lane
#pragma unroll
            for (int d = 4; d >= 1; d >>= 1) v += wp::shfl_xor(v, d);
            return wp::shfl(v, 0);
        };
        const int m0 = total(wp::popc(pl_match(rp, rf)));
        D = R.dg_a4 * m0 + R.dg_b4 * (I - m0);
        proved = D > R.dg_thr4;
#pragma unroll
        for (int t = 1; t <= 4; t++) {
            if (t > dS) break;
            // offset +t: reference row x against read base x + t; offset -t: read base x against reference row x + t
            const int m = total((wp::popc(pl_match(rf, pl_shifted(rp, rp1, t))) << 16) | wp::popc(pl_match(rp, pl_shifted(rf, rf1, t))));
            const int mp = m >> 16, mn = m & 0xffff;
            proved = proved && D > R.dg_a4 * mp + R.dg_b4 * (I - t - mp) + R.dg_c4[4 + t] &&
                     D > R.dg_a4 * mn + R.dg_b4 * (I - t - mn) + R.dg_c4[4 - t];
        }
    } else {
        const int32_t *prof = R.prof;                // [q][Ipad]: 4 x matrix[reference row][alphabet[q]]
        const int Ipad = R.Ipad;
        int acc[9];                                  // acc[s + 4]: 4 x ungapped score of read base k + s against reference row k
#pragma unroll
        for (int s = 0; s < 9; s++) acc[s] = 0;
        for (int k = lane; k < I; k += 32) {
            const int32_t *pk = prof + k;
#pragma unroll
            for (int s = -4; s <= 4; s++) {
                const int j = k + s;
                if ((s < 0 ? -s : s) <= dS && j >= 0 && j < J) acc[s + 4] += pk[(int)c[j] * Ipad];
            }
        }
#pragma unroll
        for (int s = 0; s < 9; s++)
            if ((s < 4 ? 4 - s : s - 4) <= dS)
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) acc[s] += wp::shfl_xor(acc[s], d);
        D = acc[4];
        proved = D > R.dg_thr4;
#pragma unroll
        for (int s = -4; s <= 4; s++)
            if (s != 0 && (s < 0 ? -s : s) <= dS) proved = proved && D > acc[s + 4] + R.dg_c4[s + 4];
    }
    if (!proved) return P.route == 0 ? DG_KEEP : P.route == 2 ? DG_ROUTE : route_read(R, S, D >> 2);
    // what align_narrow16 writes for an all-M traceback of I columns: op words of 32 ops, OP_NONE (3) past the end
    const int64_t slot = oslot(P, rd, r);
    if (lane < 16 && lane < P.NW) {
        const int rem = I - 32 * lane;
        P.gops[slot * P.NW + lane] = rem >= 32 ? 0ull : rem <= 0 ? ~0ull : (~0ull << (2 * rem));
    }
    if (lane == 0) P.gmeta[slot] = gmeta_pack(I, mode == 1, GM_ALIGNED);
    diag_classify(P, S, R, c, rd, r, mode == 1, cnt, w, A, R.dg_two && acgt);
    return DG_PROVED;
}

C2B_DEV void dsmem_init(const KParams &P, DSmem &S)
{
    for (int k = wp::lane(); k < 256; k += 32) S.lut[k] = P.lut[k];
    if (wp::lane() == 0) { S.pl_ref = -1; S.npop = 0; }
    wp::sync();
}

// Read x of the unit towards S.raw[b]: the 16-byte lines that hold its bytes (read byte p at S.raw[b][(address & 15) + p]),
// copied in the background while the warp works on the read before it.  A line reaching past the read buffer is copied byte by
// byte, nothing outside the buffer.  Reads longer than RG_COMBO are not copied: diag_read leaves them without looking.
C2B_DEV void diag_stage(const KParams &P, DSmem &S, int x, int b)
{
    const int64_t off = S.off[x];
    if (S.off[x + 1] - off > RG_COMBO) return;
    const uint8_t *p0 = P.reads + off, *end = P.reads + S.off[x + 1], *lim = P.reads + S.total_bytes;
    const int lane = wp::lane();
    const uint8_t *wa = p0 - ((uintptr_t)p0 & 15) + 16 * lane;
    uint8_t *dst = S.raw[b] + 16 * lane;
    if (wa >= end) return;
    if (wa >= P.reads && wa + 16 <= lim) wp::cp_async16(dst, wa);
    else for (int k = 0; k < 16; k++) if (wa + k >= P.reads && wa + k < lim) dst[k] = wa[k];
}

// warp-aggregated append of reads first + x (bit x of mask) to a list: one atomic, the reads stay in order
C2B_DEV void list_append(int32_t *list, unsigned long long *n, uint32_t mask, int64_t first)
{
    if (!mask) return;
    const int lane = wp::lane();
    unsigned long long pos = 0;
    if (lane == 0) pos = wp::fetch_add(n, (unsigned long long)wp::popc(mask));
    pos = (unsigned long long)(uint32_t)wp::shfl((int)(uint32_t)pos, 0) | ((unsigned long long)(uint32_t)wp::shfl((int)(uint32_t)(pos >> 32), 0) << 32);
    if ((mask >> lane) & 1u) list[pos + wp::popc(mask & ((1u << lane) - 1u))] = (int32_t)(first + lane);
}

// reads 32u .. 32u+31: returns the number proved, `routed` the number sent straight to tier 2; A: the warp's scalar
// accumulators (flushed by the caller)
C2B_DEV int diag_unit(const KParams &P, DSmem &S, int64_t u, ScAcc<1> &A, int &routed)
{
    const int lane = wp::lane();
    const int64_t first = 32 * u;
    const int n = P.n_reads - first < 32 ? (int)(P.n_reads - first) : 32;
    {
        const int64_t rd = first + lane;
        if (lane < n) {
            S.off[lane] = P.offsets[rd]; S.ref[lane] = P.ref_id ? P.ref_id[rd] : 0;
            S.cnt[lane] = P.count ? P.count[rd] : 1; S.qw[lane] = P.qweight ? P.qweight[rd] : S.cnt[lane];
        }
        if (lane == 0) { S.off[n] = P.offsets[first + n]; S.total_bytes = P.offsets[P.n_reads]; }
    }
    wp::sync();
#ifndef C2B_EMU
    {                                                // the unit's bytes towards L2 (about 8 KB), one request per line
        const int64_t b0 = S.off[0] & ~(int64_t)127, b1 = S.off[n];
        for (int64_t a = b0 + (int64_t)lane * 128; a < b1; a += 32 * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(P.reads + a));
    }
#endif
    uint32_t fail = 0, route = 0;
    diag_stage(P, S, 0, 0);
#pragma unroll 1
    for (int x = 0; x < n; x++) {
        const int64_t off = S.off[x];
        wp::wait_async();
        wp::sync();                                  // read x's bytes are in S.raw[x & 1]; read x + 1's go towards the other buffer
        if (x + 1 < n) diag_stage(P, S, x + 1, (x + 1) & 1);
        const int v = diag_read(P, S, first + x, S.raw[x & 1] + ((uintptr_t)(P.reads + off) & 15), (int)(S.off[x + 1] - off), S.ref[x],
                                S.cnt[x], S.qw[x], A);
        if (v != DG_PROVED) fail |= 1u << x;
        if (v == DG_ROUTE) route |= 1u << x;
        wp::sync();
    }
    list_append(P.left0, &P.wb->launch.diag_n, fail, first);   // every unproved read: CLASSIFY's list
    if (P.route) {                                   // routing: the narrow tier's list and the tier-2 list
        list_append(P.left1, &P.wb->launch.narrow_n, fail & ~route, first);
        list_append(P.left2, &P.wb->launch.tier2_n, route, first);
    }
    routed = wp::popc(route);
    return n - wp::popc(fail);
}

// The diagonal tier's loop for warp `warp` of `nwarps`: units of 32 consecutive reads strided over the warps; the warp's
// counts go to the work block once, at the end
C2B_DEV void diag_loop(const KParams &P, DSmem &S, int64_t warp, int64_t nwarps)
{
    dsmem_init(P, S);
    ScAcc<1> acc;
    sc_init(acc);
    const int64_t units = (P.n_reads + 31) / 32;
    int proved = 0, seen = 0, routed = 0;
    for (int64_t u = warp; u < units; u += nwarps) {
        int k = 0;
        proved += diag_unit(P, S, u, acc, k);
        routed += k;
        seen += P.n_reads - 32 * u < 32 ? (int)(P.n_reads - 32 * u) : 32;
        wp::sync();
    }
    sc_flush(acc, P);
    if (wp::lane() == 0 && seen) {
        WorkBlock &wb = *P.wb;
        wp::addg(&wb.diag_proved, proved); wp::addg(&wb.diag_listed, seen - proved);
        wp::addg(&wb.tier2, routed);                    // tier-2 reads: routed here, and the narrow tier's failures
        wp::addg(&wb.routed, routed); wp::addg(&wb.kept, seen - proved - routed);
        wp::addg(&wb.diag_popc, S.npop);
    }
}

}  // namespace c2b
