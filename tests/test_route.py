"""Routing in the diagonal tier (route_read): reads the narrow first tier cannot prove go straight to the wide-ring second tier.
Routing only decides which exact tier aligns a read, so every batch here runs three ways -- routing on, C2B_NO_ROUTE=1 (the
launch sequence without it) and C2B_ROUTE_ALL=1 (every unproved read routed) -- and the three must agree field by field:
records, alignments, strings, edit lists, used op words, compact outputs and the count block.  The counters must add up, and
the number of routed reads must equal a numpy restatement of the rule (DESIGN.md section 3).  The routing test keeps a read only
when it has found a path inside the narrow band that beats the narrow bound, so with routing on the narrow tier must never fail
a read of the amplicon's length.  Runs on the CPU warp emulator; the same checks run through the sm_90a library when a GPU is
present."""
import os

import numpy as np
import pytest

import parity_util as PU
import test_diag_tier as DT
from crispresso2_b200 import synth
from crispresso2_b200.engine import Engine, pack_reads
from oracle import oracle as O

MODES = (None, "C2B_NO_ROUTE", "C2B_ROUTE_ALL")
RN_DLO, RN_DHI = 17, 11                                   # the narrow tier's band (align_narrow16)
ACGT = list("ACGT")


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def emu(request):
    """the warp-emulator build; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0)
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build())


def same(a, ca, xa, b, cb, xb):
    """run_both's comparison (test_diag_tier.py) of two runs of one batch"""
    assert (a.recs == b.recs).all() and (a.alns == b.alns).all() and (ca == cb).all()
    assert ((xa.meta & 0xffffff) == (xb.meta & 0xffffff)).all() and (((xa.meta >> 24) != 0) == ((xb.meta >> 24) != 0)).all()
    cols = np.arange(a.W)[None, :] >= (a.W - a.alns[:, 0]["aln_len"].astype(np.int64))[:, None]
    assert ((a.strings[:, 0] == b.strings[:, 0]) | ~cols[:, None, :]).all()
    (ea, fa), (eb, fb) = PU.edits_canonical(a), PU.edits_canonical(b)
    assert (fa == fb).all() and (ea[fa] == eb[fb]).all()
    nw = (xa.meta.reshape(-1) & 0xffff).astype(np.int64)
    ops_a, ops_b = xa.ops.reshape(len(nw), -1), xb.ops.reshape(len(nw), -1)
    for k in range(len(nw)):
        used = (int(nw[k]) + 31) // 32
        assert (ops_a[k, :used] == ops_b[k, :used]).all(), k


def run_three(engine, refs, names, reads, go=-20, ge=-2, flags=0, matrix=None):
    """-> {mode: (diag_counts, route_counts)}; asserts that the three modes computed the same and that the counters add up"""
    m = O.make_matrix() if matrix is None else matrix
    buf, off = pack_reads(reads)
    n = len(reads)
    out = {}
    for mode in MODES:
        if mode:
            os.environ[mode] = "1"
        try:
            engine.configure(refs, names, m, go, ge, 5, 2, flags, "ACGTN", 48)
            engine.counts_reset()
            res = engine.align_packed(buf, off)
            dc, rt = engine.diag_counts(), engine.route_counts()
            cres = engine.align_packed(buf, off, compact=True, count=np.zeros(n, dtype=np.int32), qweight=np.zeros(n, dtype=np.int32))
            out[mode] = (res, engine.counts_raw(), cres, dc, rt)
        finally:
            if mode:
                os.environ.pop(mode, None)
    a, ca, xa = out[None][:3]
    for mode in MODES[1:]:
        same(a, ca, xa, *out[mode][:3])
    I = len(refs[names[0]]["sequence"])
    for mode in MODES:
        (proved, listed, _), (routed, kept) = out[mode][3:]
        if proved + listed:                               # the diagonal tier ran
            assert proved + listed == n and kept + routed == listed, (mode, out[mode][3:])
    assert out["C2B_NO_ROUTE"][4][0] == 0
    (proved, listed, tier2), (routed, kept) = out[None][3:]
    if proved + listed and all(len(r) == I for r in reads):
        assert tier2 == routed                      # tier-2 reads: routed ones only, a kept read has a path in the band
                                                    # that beats the narrow bound
    assert out["C2B_ROUTE_ALL"][4][0] >= routed
    return {mode: out[mode][3:] for mode in MODES}


# ------------------------------------------------------------------------------------------------ the rule, restated
def route_rule(reads, ref, go=-20, ge=-2, matrix=None, alphabet="ACGTN"):
    """-> (proved, routed) over `reads` against one amplicon: the diagonal tier's proof rule (test_diag_tier.rule_count)
    and the routing test of route_read, vectorised over the reads"""
    m = O.make_matrix() if matrix is None else matrix
    seq = ref["sequence"]
    I = len(seq)
    gi = np.asarray(ref["gap_incentive"], dtype=np.int64)
    nq = len(alphabet)
    rows = np.array([[m[ord(seq[i]), ord(q)] for i in range(I)] for q in alphabet], dtype=np.int64)     # [q][i]
    rcode = np.array([alphabet.index(c) if c in alphabet else 255 for c in seq])
    smax, gp, gmin = int(rows.max()), max(int(gi.max()), 0), int(gi.min())
    dg_ok = go <= ge <= 0 and gmin >= 0 and 2 * (ge + gp) <= smax and I >= 2 and I <= 256
    if not dg_ok:
        return 0, 0
    thr = max(smax * (I - 1) + go + ge + 2 * gp, go * I * I + max(smax, 0) * I + 2 * I * gp)
    edge = lambda t: smax * (I - t) + t * (2 * ge + gp) + gp
    S = 0
    while S < 4 and S + 1 < I and edge(S + 1) > thr:
        S += 1
    if S + 1 < I:
        thr = max(thr, edge(S + 1))
    c4 = {s: 2 * ge * abs(s) + int(gi[0]) + (int(gi[I - s]) if s > 0 else abs(s) * int(gi[I])) for s in range(-S, S + 1) if s}
    # routing constants (c2b_configure)
    nq4 = min(nq, 4)
    matched = np.zeros((nq, I), dtype=bool)
    for i in range(I):
        if rcode[i] < nq4:
            matched[rcode[i], i] = True
    rm, rx = int(rows[matched].min()), int(rows[~matched].min())
    gmax, gsum = int(gi.max()), int(gi.sum())
    rthr = max(smax * (I - d - 1) + (d + 1) * (ge + gmax) + (d + 1) * ge + gsum for d in (RN_DHI, RN_DLO) if d + 1 <= I)
    offs = [s for s in range(-16, 16) if s and abs(s) < I and (abs(s) <= RN_DLO if s < 0 else abs(s) <= RN_DHI)]
    cost = {s: go + (abs(s) - 1) * ge + (abs(s) * (ge + int(gi[I])) if s < 0 else abs(s) * ge + int(gi[I - abs(s)])) + rx * (I - abs(s))
            for s in offs}
    # reads of the amplicon's length, every base in the alphabet, one strand
    params = O.Params()
    codes, keep_idx, routed = [], [], 0
    for k, read in enumerate(reads):
        if len(read) != I:
            continue
        if any(ch not in alphabet for ch in read):
            routed += 1
            continue
        strand = O._strand_choice(params, read, ref)
        if strand == "both":
            routed += 1
            continue
        s_read = read if strand == "fw" else DT.rc(read)
        codes.append([alphabet.index(ch) for ch in s_read])
        keep_idx.append(k)
    if not codes:
        return 0, routed
    R = np.array(codes, dtype=np.int64)                                           # [n][I]
    n = len(R)
    ii = np.arange(I)
    sc = rows[R, ii[None, :]]                                                     # score of read column i on row i
    D = sc.sum(1)

    def diag(s):                                                                  # sum_i s(i, i + s)
        lo, hi = max(0, -s), min(I, I - s)
        return rows[R[:, lo + s:hi + s], ii[None, lo:hi]].sum(1)

    proved = D > thr
    for s, c in c4.items():
        proved &= D > diag(s) + c
    todo = ~proved & (D <= rthr)                                                  # D beating the narrow bound: kept
    if not offs:
        return int(proved.sum()), routed + int(todo.sum())
    valid_r = R < 4
    valid_f = rcode < 4
    m0 = valid_r & valid_f[None, :] & (R == rcode[None, :])
    nb = (I + 31) // 32
    best_val, best = np.full(n, -(1 << 62), dtype=np.int64), {}
    for s in offs:
        t = abs(s)
        ms = np.zeros((n, I), dtype=bool)
        if s < 0:                                                                 # read x against reference x + t
            ms[:, :I - t] = valid_r[:, :I - t] & valid_f[None, t:] & (R[:, :I - t] == rcode[None, t:])
        else:                                                                     # reference x against read x + t
            ms[:, :I - t] = valid_f[None, :I - t] & valid_r[:, t:] & (rcode[None, :I - t] == R[:, t:])
        m0s = m0.copy()
        m0s[:, I - t:] = False
        c0, cs = np.cumsum(m0s, 1), np.cumsum(ms, 1)
        mst = cs[:, -1]
        ends = np.minimum(32 * np.arange(1, nb + 1), I) - 1                      # block ends p = 32 (b + 1), last index below
        P = c0[:, ends] - cs[:, ends]
        bb = P.argmax(1) + 1                                                      # first block end attaining the best
        val = rm * (mst + P.max(1)) - rx * (mst + P.max(1)) + cost[s]
        better = val > best_val                                                   # offsets in increasing order: first wins ties
        best_val = np.where(better, val, best_val)
        best[s] = (bb, c0, cs, mst)
        if s == offs[0]:
            choice = np.full(n, s)
        choice = np.where(better, s, choice)
    e = np.full(n, -(1 << 62), dtype=np.int64)
    for s in offs:
        sel = choice == s
        if not sel.any():
            continue
        t = abs(s)
        bb, c0, cs, mst = best[s]
        cz = np.concatenate([np.zeros((n, 1), np.int64), c0], 1)                  # M0[0, p) for p = 0..I
        csz = np.concatenate([np.zeros((n, 1), np.int64), cs], 1)
        F = cz + mst[:, None] - csz                                               # F(p), p = 0..I
        p = np.arange(I + 1)
        w0 = bb - 1
        inwin = (p[None, :] >= 32 * w0[:, None]) & (p[None, :] <= 32 * w0[:, None] + 64) & (p[None, :] >= 1) & (p[None, :] <= I - t)
        imul = 1 if s < 0 else t
        inc = np.concatenate([gi[:I], [0]])
        v = (rm - rx) * F + imul * inc[None, :] + cost[s]
        v = np.where(inwin, v, -(1 << 62)).max(1)
        e = np.where(sel, v, e)
    routed += int((todo & ~(e > rthr)).sum())
    return int(proved.sum()), routed


def check_rule(counts, reads, ref, **kw):
    proved, routed = route_rule(reads, ref, **kw)
    (dp, _, _), (dr, _) = counts[None]
    assert (dp, dr) == (proved, routed)


# ---------------------------------------------------------------------------------------------------------- tests
def setup(I=250, seed=42, **kw):
    amp = synth.random_amplicon(np.random.default_rng(seed), I)
    ref = synth.amplicon_setup(amp, **kw)
    return amp, ref, {"Reference": ref}, ["Reference"]


def pad(rng, s, I):
    return (s + "".join(rng.choice(ACGT, max(0, I - len(s)))))[:I]


def test_bench_mix(emu):
    rng = np.random.default_rng(5)
    amp, ref, refs, names = setup(guide_start=110)
    reads = [r.tobytes().decode() for r in synth.synth_reads_fast(rng, amp, 2048, 250, cut=ref["cut_point"])]
    counts = run_three(emu, refs, names, reads)
    (proved, listed, _), (routed, kept) = counts[None]
    assert routed > 0 and kept > 0 and counts["C2B_ROUTE_ALL"][1] == (listed, 0)
    check_rule(counts, reads, ref)
    PU.check_against_oracle(emu, refs, names, O.Params(), reads[:256], O.make_matrix())


def test_indels_at_the_cut_and_block_edges(emu):
    rng = np.random.default_rng(7)
    amp, ref, refs, names = setup()
    I, cut = len(amp), ref["cut_point"]
    reads = []
    for p in (cut + 1, 3, 20, I - 30, I - 12, 30, 31, 32, 33, 62, 63, 64, 65):
        reads += [pad(rng, amp[:p] + amp[p + d:], I) for d in range(1, 25)]
        reads += [(amp[:p] + "".join(rng.choice(ACGT, k)) + amp[p:])[:I] for k in range(1, 13)]
    counts = run_three(emu, refs, names, reads)
    assert counts[None][1][0] > 0 and counts[None][1][1] > 0
    check_rule(counts, reads, ref)


def test_substitution_counts_around_the_bound(emu):
    rng = np.random.default_rng(8)
    amp, ref, refs, names = setup()
    reads = DT.edited_reads(rng, amp, [ns for ns in range(15) for _ in range(6)])
    reads += [pad(rng, amp[:126] + amp[130:], len(amp))] * 2       # a deletion of 4 beside them
    counts = run_three(emu, refs, names, reads)
    check_rule(counts, reads, ref)
    PU.check_against_oracle(emu, refs, names, O.Params(), reads, O.make_matrix())


def test_n_bases_other_symbols_both_strands_and_reverse_complements(emu):
    rng = np.random.default_rng(9)
    while True:                                           # an amplicon whose own seed test is one-sided
        amp, ref, refs, names = setup(seed=int(rng.integers(1 << 30)))
        if O._strand_choice(O.Params(), amp, ref) == "fw":
            break
    I, cut = len(amp), ref["cut_point"]
    base = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 48, I, sub_rate=0.01, cut=cut)]
    withn = [r[:p] + "N" + r[p + 1:] for r, p in zip(base[:24], rng.integers(0, I, 24))]
    withn += [amp[:cut - 3] + "NNNN" + amp[cut + 1:], pad(rng, amp[:cut] + amp[cut + 9:cut + 20] + "N" + amp[cut + 21:], I)]
    both = [amp[:40] + "".join(rng.choice(ACGT, I - 80)) + amp[-40:] for _ in range(6)]
    reads = base + withn + both + [DT.rc(r) for r in base[:24] + withn[:8]]
    counts = run_three(emu, refs, names, reads)
    check_rule(counts, reads, ref)
    PU.check_against_oracle(emu, refs, names, O.Params(), reads, O.make_matrix())
    odd = reads[:40] + [amp[:100] + "X" + amp[101:]] + reads[40:60]           # a symbol outside the alphabet
    counts = run_three(emu, refs, names, odd)
    check_rule(counts, odd, ref)


@pytest.mark.parametrize("kind", ["tandem", "homopolymer"])
def test_repeats_where_the_shift_is_ambiguous(emu, kind):
    rng = np.random.default_rng(10)
    amp = "AC" * 125 if kind == "tandem" else "".join(c * 25 for c in "ACGTAGCTAC")
    ref = synth.amplicon_setup(amp, guide_start=100, seed_count=5)
    refs, names = {"Reference": ref}, ["Reference"]
    I, cut = len(amp), ref["cut_point"]
    reads = DT.edited_reads(rng, amp, [1, 2, 4, 8, 12] * 4)
    for d in (1, 2, 5, 8, 9, 10, 16):
        reads += [pad(rng, amp[:cut] + amp[cut + d:], I), pad(rng, amp[:60] + amp[60 + d:], I)]
    for k in (1, 2, 3, 9, 10, 11):
        reads += [(amp[:cut] + amp[cut - k:cut] + amp[cut:])[:I], (amp[:cut] + "G" * k + amp[cut:])[:I]]
    counts = run_three(emu, refs, names, reads)
    check_rule(counts, reads, ref)
    PU.check_against_oracle(emu, refs, names, O.Params(), reads, O.make_matrix())


@pytest.mark.parametrize("I", [187, 200, 233, 255])
def test_amplicon_lengths_off_the_word_size(emu, I):
    rng = np.random.default_rng(I)
    amp, ref, refs, names = setup(I=I, seed=I, guide_start=I // 2 - 10)
    reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 200, I, sub_rate=0.01, cut=ref["cut_point"])]
    reads += [pad(rng, amp[:I - 20] + amp[I - 20 + d:], I) for d in range(1, 12)]
    counts = run_three(emu, refs, names, reads)
    check_rule(counts, reads, ref)
    PU.check_against_oracle(emu, refs, names, O.Params(), reads[:96], O.make_matrix())


@pytest.mark.parametrize("matrix,go,ge,gi", [(O.make_matrix(10, -8, -4, -2), -40, -4, 2), (O.make_matrix(), -5, -5, 1),
                                             (O.make_matrix(), -10, -3, 2)])
def test_scoring(emu, matrix, go, ge, gi):
    rng = np.random.default_rng(11 + gi)
    amp, ref, refs, names = setup(gap_incentive_value=gi)
    reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 256, 250, sub_rate=0.01, cut=ref["cut_point"])]
    counts = run_three(emu, refs, names, reads, go=go, ge=ge, matrix=matrix)
    assert counts[None][0][0] > 0
    check_rule(counts, reads, ref, go=go, ge=ge, matrix=matrix)
    P = O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge)
    PU.check_against_oracle(emu, refs, names, P, reads[:96], matrix)


@pytest.mark.parametrize("n", [16, 17, 33, 50, 71, 100])
def test_batch_sizes_and_partial_units(emu, n):
    rng = np.random.default_rng(100 + n)
    amp, ref, refs, names = setup()
    reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, n, 250, sub_rate=0.01, del_frac=0.4, ins_frac=0.2,
                                                             cut=ref["cut_point"])]
    counts = run_three(emu, refs, names, reads)
    check_rule(counts, reads, ref)


def test_every_read_routed_and_none_routed(emu):
    rng = np.random.default_rng(12)
    amp, ref, refs, names = setup()
    I, cut = len(amp), ref["cut_point"]
    far = [pad(rng, amp[:cut] + amp[cut + d:], I) for d in rng.integers(12, 21, 40)]
    counts = run_three(emu, refs, names, far)
    (proved, listed, _), (routed, kept) = counts[None]
    assert (proved, listed, routed, kept) == (0, 40, 40, 0)
    near = DT.edited_reads(rng, amp, [3, 4, 5, 6, 7] * 8)
    near = [r for r in near if O._strand_choice(O.Params(), r, ref) == "fw"][:32]     # substitutions in seeds: both strands
    counts = run_three(emu, refs, names, near)
    (proved, listed, _), (routed, kept) = counts[None]
    assert (proved, listed, routed, kept) == (0, 32, 0, 32)


def test_rule_matches_on_a_large_bench_batch(emu):
    """64 Ki bench-mix reads (8 Ki on the emulator) with routing on: the device's routed count equals the restated rule's"""
    rng = np.random.default_rng(13)
    amp, ref, refs, names = setup()
    n = 1 << 13 if "emu" in str(emu.lib_path) else 1 << 16
    reads = [r.tobytes().decode() for r in synth.synth_reads_fast(rng, amp, n, 250, cut=ref["cut_point"])]
    buf, off = pack_reads(reads)
    emu.configure(refs, names, O.make_matrix(), -20, -2, 5, 2, 0, "ACGTN", 48)
    emu.counts_reset()
    emu.align_packed(buf, off, strings=False, edits=False)
    (proved, listed, tier2), (routed, kept) = emu.diag_counts(), emu.route_counts()
    assert proved + listed == len(reads) and routed + kept == listed and tier2 == routed
    assert (proved, routed) == route_rule(reads, ref)
    assert routed > len(reads) // 10
