// c2b_annotate.cuh -- the read annotations of --fastq_output / --bam_output, built on the device from the compact batch results.
//
// Replaces the per-read annotation code of process_fastq_write_out (CRISPRessoCORE.py:2302-2343) and
// process_single_fastq_write_bam_out (:2399-2497): for every unique read, the text
//   " ALN=<names> ALN_SCORES=<scores> ALN_DETAILS=<name,aln_seq,aln_ref,score per reference> CLASS=<class_name>
//    MODS=D<n>;I<n>;S<n> DEL=<start(size)> INS=<start(size+BASES)> SUB=<pos> ALN_REF=<aligned refs> ALN_SEQ=<aligned reads>"
// (lists of one reference joined by ';', references by '&'), the short " ALN=NA ALN_SCORES=.. ALN_DETAILS=.." of a read that
// did not align, and for the first aligned reference the SAM CIGAR (CRISPRessoShared.CIGAR_LOOKUP + unexplode_cigar,
// CRISPRessoShared.py:426-434, 561-582), flag and MAPQ.
//
// One warp per unique read.  The aligned strings of every (read, reference) slot are spelled from the op stream by the whole
// warp (lane l holds op word l: columns 32l..32l+31 counted from the right; a shuffle scan of the per-word base counts gives
// every column its read / reference index); the short fields are formatted by every lane alike (warp-uniform control flow,
// lane 0 stores).  The same routine runs twice: with no output buffer it only counts bytes (size pass), then, after a scan of
// the sizes, it writes (write pass).
//
// Compiled by nvcc for sm_90a (c2b_engine.cu) and by g++ against the warp emulator (tests/emu/): nothing here needs CUB.
#pragma once

namespace c2b {
namespace ann {

struct AParams {
    const uint8_t *reads; const int64_t *roff; int64_t n;      // unique reads of this chunk
    const int32_t *bidx;                                       // per unique: its index in the batch arrays below, -1 = not in the batch
    int32_t R, NW, cap; uint32_t flags;                        // slots per read, op words per slot, edit-list cap, C2B_F_LEGACY_INS
    const c2b_read_rec *recs; const c2b_aln_rec *alns; const uint64_t *ops; const uint32_t *meta; const c2b_edit *edits;
    const uint32_t *amask;                                     // per batch read: slots listed in aln_ref_names (0 = not aligned)
    const int16_t *aname;                                      // per batch read: name id of the one listed slot, -1 = the slot's own name
    const int32_t *label;                                      // per batch read: class_name id
    const char *names; const int32_t *name_off; const uint8_t *name_rev;   // name table (refs[name]['aln_strand'] == '-')
    const char *labels; const int32_t *label_off;
    const char *refseq; const int32_t *ref_off;                // the R reference sequences
    const uint8_t *comp;                                       // byte -> complement (reads aligned as their reverse complement)
    int64_t *ann_len, *cig_len;                                // size pass
    const int64_t *ann_off, *cig_off;                          // write pass: exclusive scans of the sizes (n + 1)
    char *ann, *cig; uint8_t *flag; int32_t *mapq; int16_t *first;
};

struct Out { char *p; int64_t n; };

C2B_DEV void put(Out &o, char c)
{
    if (o.p && wp::lane() == 0) o.p[o.n] = c;
    o.n++;
}

C2B_DEV void put_str(Out &o, const char *s, int len)       // all lanes
{
    if (o.p) for (int i = wp::lane(); i < len; i += 32) o.p[o.n + i] = s[i];
    o.n += len;
}

C2B_DEV void put_uint(Out &o, uint64_t v)
{
    char d[20];
    int k = 0;
    do { d[k++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (k) put(o, d[--k]);
}

C2B_DEV void put_int(Out &o, int64_t v)
{
    if (v < 0) { put(o, '-'); v = -v; }
    put_uint(o, (uint64_t)v);
}

// str(k / 1000.0) for the scores round(100 * m / n, 3) = k / 1000 (Python's shortest repr: the decimal with trailing zeros
// trimmed, at least one digit after the point)
C2B_DEV void put_score(Out &o, int32_t k)
{
    if (k < 0) { put(o, '-'); k = -k; }
    put_uint(o, (uint64_t)(k / 1000));
    put(o, '.');
    int f = k % 1000, nd = 3;
    if (f == 0) { put(o, '0'); return; }
    while (f % 10 == 0) { f /= 10; nd--; }
    const int p10[3] = {1, 10, 100};
    for (int d = nd - 1; d >= 0; d--) put(o, (char)('0' + (f / p10[d]) % 10));
}

C2B_DEV int op_at(uint64_t w, int t) { return (int)((w >> (2 * t)) & 3ull); }

// exclusive prefix over lanes of v (lane order = columns from the right)
C2B_DEV int lane_excl_scan(int v)
{
    int s = v;
    for (int d = 1; d < 32; d <<= 1) { const int u = wp::shfl_up(s, d); if (wp::lane() >= d) s += u; }
    return s - v;
}

// Aligned read (which = 0) or reference (which = 1) string of one slot, left to right, n columns (Align.pyx:422-432):
// column q from the right consumes read / reference when its op is not a gap on that side; the idx-th consuming column from
// the right holds read[rlen - 1 - idx] (forward strand), comp[read[idx]] (reverse complement) or ref[ilen - 1 - idx].
C2B_DEV void spell(Out &o, const uint64_t *ops, int n, int which, const uint8_t *read, int rlen, int strand, const char *ref,
                   int ilen, const uint8_t *comp)
{
    const int l = wp::lane();
    const uint64_t w = (32 * l < n) ? ops[l] : 0ull;
    const int gap = which ? OP_I : OP_J;
    int cnt = 0;
    for (int t = 0; t < 32 && 32 * l + t < n; t++) cnt += op_at(w, t) != gap;
    int idx = lane_excl_scan(cnt);
    if (o.p)
        for (int t = 0; t < 32 && 32 * l + t < n; t++) {
            const int q = 32 * l + t;
            char c = '-';
            if (op_at(w, t) != gap) {
                c = which ? ref[ilen - 1 - idx] : strand ? (char)comp[read[idx]] : (char)read[rlen - 1 - idx];
                idx++;
            }
            o.p[o.n + (n - 1 - q)] = c;
        }
    o.n += n;
}

// ref_positions.index(a) (COREResources.pyx:105-133): the column, from the left, that holds reference base a; -1 if none
C2B_DEV int ref_column(const uint64_t *ops, int n, int ilen, int a)
{
    const int l = wp::lane();
    const uint64_t w = (32 * l < n) ? ops[l] : 0ull;
    int cnt = 0;
    for (int t = 0; t < 32 && 32 * l + t < n; t++) cnt += op_at(w, t) != OP_I;
    int idx = lane_excl_scan(cnt);
    const int want = ilen - 1 - a;                              // reference-consuming columns to its right
    int q = -1;
    if (want >= idx && want < idx + cnt)
        for (int t = 0; t < 32 && 32 * l + t < n; t++)
            if (op_at(w, t) != OP_I) { if (idx == want) { q = 32 * l + t; break; } idx++; }
    const uint32_t b = wp::ballot(q >= 0);
    if (!b) return -1;
    q = wp::shfl(q, wp::ffs(b) - 1);
    return n - 1 - q;
}

// the listed slots (aln_ref_names order) of one batch read
C2B_DEV int listed(const AParams &P, int64_t k, int *slot, int *name)
{
    uint32_t m = P.amask[k];
    int c = 0;
    while (m) {
        const int s = wp::ffs(m) - 1;
        m &= m - 1;
        slot[c] = s; name[c] = P.aname[k] >= 0 ? P.aname[k] : s; c++;
    }
    return c;
}

C2B_DEV void put_name(Out &o, const AParams &P, int id) { put_str(o, P.names + P.name_off[id], P.name_off[id + 1] - P.name_off[id]); }

C2B_DEV int slot_cols(const AParams &P, int64_t k, int s)
{
    const uint32_t m = P.meta[k * P.R + s];
    return (m >> 24) ? (int)(m & 0xffffu) : 0;
}

// copy of n bytes written earlier in this annotation (all lanes; the caller synchronised the warp)
C2B_DEV void put_copy(Out &o, int64_t from, int n)
{
    if (o.p) for (int i = wp::lane(); i < n; i += 32) o.p[o.n + i] = o.p[from + i];
    o.n += n;
}

// one unique read: annotation text (+ CIGAR / flag / MAPQ of the first listed slot)
template <bool WRITE>
C2B_DEV void annotate_one(const AParams &P, int64_t u)
{
    Out o{WRITE ? P.ann + P.ann_off[u] : nullptr, 0};
    const int64_t k = P.bidx[u];
    const char *na = " ALN=NA";
    if (k < 0) {                                                // outside the engine's contract: no scores, no details
        put_str(o, na, 7);
        put_str(o, " ALN_SCORES= ALN_DETAILS=", 25);
        if (!WRITE) { if (wp::lane() == 0) { P.ann_len[u] = o.n; P.cig_len[u] = 0; } }
        else if (wp::lane() == 0) { P.flag[u] = 255; P.mapq[u] = 0; P.first[u] = -1; }
        return;
    }
    const int R = P.R;
    const uint8_t *read = P.reads + P.roff[u];
    const int rlen = (int)(P.roff[u + 1] - P.roff[u]);
    int slot[32], name[32];
    const int nl = listed(P, k, slot, name);
    if (nl == 0) put_str(o, na, 7);
    else {
        put_str(o, " ALN=", 5);
        for (int x = 0; x < nl; x++) { if (x) put(o, '&'); put_name(o, P, name[x]); }
    }
    put_str(o, " ALN_SCORES=", 12);
    for (int r = 0; r < R; r++) { if (r) put(o, '&'); put_score(o, P.alns[k * R + r].score_milli); }
    put_str(o, " ALN_DETAILS=", 13);
    int64_t det[32];                                            // where slot r's aligned read starts in this annotation
    for (int r = 0; r < R; r++) {
        if (r) put(o, '&');
        put_name(o, P, r);
        put(o, ',');
        const int n = slot_cols(P, k, r);
        const int strand = (int)((P.meta[k * R + r] >> 16) & 1u);
        const uint64_t *ops = P.ops + (k * R + r) * P.NW;
        const char *ref = P.refseq + P.ref_off[r];
        const int ilen = P.ref_off[r + 1] - P.ref_off[r];
        det[r] = o.n;
        spell(o, ops, n, 0, read, rlen, strand, ref, ilen, P.comp);
        put(o, ',');
        spell(o, ops, n, 1, read, rlen, strand, ref, ilen, P.comp);
        put(o, ',');
        put_score(o, P.alns[k * R + r].score_milli);
    }
    wp::sync();                                                 // the spelled strings are read back below
    if (nl) {
        const bool legacy = (P.flags & C2B_F_LEGACY_INS) != 0;
        put_str(o, " CLASS=", 7);
        const int lb = P.label[k];
        put_str(o, P.labels + P.label_off[lb], P.label_off[lb + 1] - P.label_off[lb]);
        put_str(o, " MODS=", 6);
        for (int x = 0; x < nl; x++) {
            const c2b_aln_rec &a = P.alns[k * R + slot[x]];
            const c2b_edit *ed = P.edits + (k * R + slot[x]) * P.cap;
            int64_t dn = a.deletion_n, in = a.insertion_n;
            if (legacy) {                                       // COREResources.pyx:262, 297: sums of the window sizes
                dn = 0; in = 0;
                for (int e = 0; e < a.n_edits; e++) {
                    if (!ed[e].in_window) continue;
                    if (ed[e].type == 3) dn += (int)ed[e].b - (int)ed[e].a + (int)ed[e].base - 2;
                    else if (ed[e].type == 2) in += ed[e].b;
                }
            }
            if (x) put(o, '&');
            put(o, 'D'); put_int(o, dn); put_str(o, ";I", 2); put_int(o, in); put_str(o, ";S", 2); put_int(o, a.substitution_n);
        }
        for (int f = 0; f < 3; f++) {                           // DEL, INS, SUB
            put_str(o, f == 0 ? " DEL=" : f == 1 ? " INS=" : " SUB=", 5);
            for (int x = 0; x < nl; x++) {
                const int s = slot[x];
                const c2b_aln_rec &a = P.alns[k * R + s];
                const c2b_edit *ed = P.edits + (k * R + s) * P.cap;
                if (x) put(o, '&');
                bool any = false;
                for (int e = 0; e < a.n_edits; e++) {
                    const c2b_edit E = ed[e];
                    if (!E.in_window || E.type != (f == 0 ? 3 : f == 1 ? 2 : 1)) continue;
                    if (any) put(o, ';');
                    any = true;
                    put_int(o, E.a);
                    if (f == 2) continue;
                    put(o, '(');
                    if (f == 0) put_int(o, legacy ? (int)E.b - (int)E.a + (int)E.base - 2 : (int)E.b - (int)E.a);
                    else {
                        // aln_seq[c + 1 : c + 1 + size] with c = ref_positions.index(start) (CRISPRessoCORE.py:2432-2436)
                        put_int(o, E.b);
                        put(o, '+');
                        const int n = slot_cols(P, k, s);
                        const int ilen = P.ref_off[s + 1] - P.ref_off[s];
                        const int c = ref_column(P.ops + (k * R + s) * P.NW, n, ilen, E.a);
                        const int lo = c + 1, hi = lo + (int)E.b < n ? lo + (int)E.b : n;
                        if (hi > lo) put_copy(o, det[s] + lo, hi - lo);
                    }
                    put(o, ')');
                }
            }
        }
        put_str(o, " ALN_REF=", 9);
        for (int x = 0; x < nl; x++) { if (x) put(o, '&'); const int n = slot_cols(P, k, slot[x]); put_copy(o, det[slot[x]] + n + 1, n); }
        put_str(o, " ALN_SEQ=", 9);
        for (int x = 0; x < nl; x++) { if (x) put(o, '&'); put_copy(o, det[slot[x]], slot_cols(P, k, slot[x])); }
    }
    // CIGAR of the first listed slot: runs of M / I (gap in the reference) / D (gap in the read) from the left; elements in
    // reverse order when refs[first]['aln_strand'] == '-' (CRISPRessoCORE.py:2462-2467)
    Out g{WRITE ? P.cig + P.cig_off[u] : nullptr, 0};
    if (nl) {
        const int s = slot[0], n = slot_cols(P, k, s);
        const bool rev = P.name_rev[name[0]] != 0;
        const uint64_t *ops = P.ops + (k * R + s) * P.NW;
        const int64_t total = WRITE ? P.cig_off[u + 1] - P.cig_off[u] : 0;
        int run = 0, prev = -1;
        for (int c = 0; c <= n; c++) {
            const int q = n - 1 - c;
            const int op = c < n ? op_at(ops[q >> 5], q & 31) : -1;
            if (op == prev) { run++; continue; }
            if (prev >= 0) {
                const char ch = prev == OP_M ? 'M' : prev == OP_I ? 'I' : 'D';
                if (rev && WRITE) {                             // element written right to left from the end
                    int len = 1; for (int v = run; v >= 10; v /= 10) len++;
                    Out h{g.p, total - g.n - (len + 1)};
                    put_uint(h, (uint64_t)run); put(h, ch);
                    g.n += len + 1;
                } else { put_uint(g, (uint64_t)run); put(g, ch); }
            }
            prev = op; run = 1;
        }
    }
    if (!WRITE) { if (wp::lane() == 0) { P.ann_len[u] = o.n; P.cig_len[u] = g.n; } }
    else if (wp::lane() == 0) {
        if (nl) {
            const int strand = (int)((P.meta[k * R + slot[0]] >> 16) & 1u);
            P.flag[u] = (uint8_t)((strand ? 16 : 0) ^ (P.name_rev[name[0]] ? 16 : 0));
            P.mapq[u] = P.recs[k].best_score_milli / 1000;        // str(int(best_match_score))
            P.first[u] = (int16_t)name[0];
        } else { P.flag[u] = 255; P.mapq[u] = 0; P.first[u] = -1; }
    }
}

// exclusive scans of the two size arrays into ann_off / cig_off (one warp: lane l sums a contiguous segment, a shuffle scan
// of the 32 segment sums, then every lane writes its segment's prefixes)
C2B_DEV void scan_sizes(const int64_t *len, int64_t *off, int64_t n)
{
    const int l = wp::lane();
    const int64_t seg = (n + 31) / 32, a = l * seg < n ? l * seg : n, b = a + seg < n ? a + seg : n;
    int64_t s = 0;
    for (int64_t i = a; i < b; i++) s += len[i];
    int64_t pre = 0, tot = 0;
    for (int j = 0; j < 32; j++) {                              // 64-bit sums through two 32-bit shuffles
        const uint32_t lo = wp::shflu((uint32_t)(uint64_t)s, j), hi = wp::shflu((uint32_t)((uint64_t)s >> 32), j);
        const int64_t v = (int64_t)(((uint64_t)hi << 32) | lo);
        if (j < l) pre += v;
        tot += v;
    }
    for (int64_t i = a; i < b; i++) { off[i] = pre; pre += len[i]; }
    if (l == 0) off[n] = tot;
}

}  // namespace ann
}  // namespace c2b

#ifndef C2B_EMU
__global__ void __launch_bounds__(256) c2b_annotate_size_kernel(const __grid_constant__ c2b::ann::AParams P)
{
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < P.n; u += nw) c2b::ann::annotate_one<false>(P, u);
}
__global__ void __launch_bounds__(256) c2b_annotate_write_kernel(const __grid_constant__ c2b::ann::AParams P)
{
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < P.n; u += nw) c2b::ann::annotate_one<true>(P, u);
}
__global__ void __launch_bounds__(32) c2b_annotate_scan_kernel(const int64_t *ann_len, int64_t *ann_off, const int64_t *cig_len,
                                                              int64_t *cig_off, int64_t n)
{
    c2b::ann::scan_sizes(ann_len, ann_off, n);
    c2b::ann::scan_sizes(cig_len, cig_off, n);
}
#endif
