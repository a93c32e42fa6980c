"""The engine against the oracle over the scoring space: substitution matrices other than EDNAFULL, gap pairs and gap incentive
profiles, placed on both sides of the host's admission rules for the exact shortcuts (DESIGN.md sections 3 and 6):

  pk_maxJ  the packed 16-bit DP (largest read length whose biased scores fit 16 bits)
  rg_ok    the 72-slot ring and the 36-slot narrow tier (ring_bound decreasing in the number of gap columns)
  dg_ok    the diagonal tier, with dg_S exactly scored offset diagonals, the bound dg_thr and the edge-run costs dg_c(s)

`admission()` restates those rules in numpy.  It is not the proof: it builds reads on both sides of each edge and says which
path must have run, which the path counters then confirm, so that a test meant for a shortcut cannot quietly exercise only
the fallback.  Every batch goes through the oracle and is compared field by field with the same batch with the shortcut off.

Also: scores whose tagged int32 DP values (4 * score + tag) could wrap must be refused (C2B_E_LIMIT), never aligned
differently from the reference, which keeps raw scores in a C int.

Runs on the CPU warp emulator; with -m gpu the same checks run through the sm_90a library with larger batches."""
import itertools
import os
import zlib

import numpy as np
import pytest

import parity_util as PU
import test_diag_tier as DT
from crispresso2_b200 import _lib, align, synth
from crispresso2_b200.engine import Engine, EngineError, pack_reads
from oracle import oracle as O

ALPHA = "ACGTN"
MAX_READ_LEN, PK_MAX_ALN2, PK_OFF = 512, 1024, 512
MATRIX_FILE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scoring_nuc.matrix")


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def eng(request):
    """(engine, batch scale): the warp-emulator build with small batches; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0), 4
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build()), 1


def ednafull():
    return O.make_matrix()


def asym(base=None, **cells):
    """a copy of `base` (EDNAFULL) with cells given as ref_read=score, e.g. A_C=-3"""
    m = np.array(ednafull() if base is None else base, dtype=np.int64)
    for k, v in cells.items():
        a, b = k.split("_")
        m[ord(a), ord(b)] = v
    return m


# ------------------------------------------------------------------------------------------------ the host's rules, restated
def admission(matrix, seq, gi, go, ge):
    """The per-reference admission rules of c2b_configure: packed path, ring, diagonal tier."""
    I = len(seq)
    rows = np.array([[matrix[ord(seq[i]), ord(q)] for i in range(I)] for q in ALPHA], dtype=np.int64)
    gi = np.asarray(gi, dtype=np.int64)
    smin, smax, gmin, gmax = int(rows.min()), int(rows.max()), int(gi.min()), int(gi.max())
    beta = -ge
    pk = (go <= ge <= 0 and gmin >= 0 and gmax <= 64 and smin + 2 * beta >= 0 and smax + 2 * beta <= 1000 and go - ge > -1900
          and 4 * (PK_OFF + go - ge) > 256 + 4 * gmax + 3 + 64)
    pk_maxJ = 0
    if pk:
        for J in range(1, MAX_READ_LEN + 1):
            if I + J > PK_MAX_ALN2 or 4 * ((smax + 2 * beta) * min(I, J) + gmax * (I + J + 2) + PK_OFF) + 3 > 32000:
                break
            pk_maxJ = J
    rg_ok = pk_maxJ > 0 and I <= 256 and smax >= 0 and 2 * ge + gmax <= smax and int(gi.sum()) < (1 << 24)
    gp = max(gmax, 0)
    thr = max(smax * (I - 1) + go + ge + 2 * gp, go * I * I + max(smax, 0) * I + 2 * I * gp)

    def edge(t):
        return smax * (I - t) + t * (2 * ge + gp) + gp
    S = 0
    while S < 4 and S + 1 < I and edge(S + 1) > thr:
        S += 1
    if S + 1 < I:
        thr = max(thr, edge(S + 1))
    thr = max(thr, -(1 << 28))
    dg_ok = rg_ok and go <= ge <= 0 and gmin >= 0 and 2 * (ge + gp) <= smax and I >= 2 and thr < (1 << 28)
    c = {s: 2 * ge * abs(s) + int(gi[0]) + (int(gi[I - s]) if s > 0 else abs(s) * int(gi[I])) for s in range(-S, S + 1) if s}
    return dict(pk_maxJ=pk_maxJ, rg_ok=rg_ok, dg_ok=dg_ok, S=S, thr=thr, c=c, smax=smax, smin=smin, gmax=gmax, gmin=gmin)


def diag_score(matrix, amp, read, s=0):
    """exact ungapped score of offset diagonal s (read base i + s against reference base i)"""
    I = len(amp)
    return sum(int(matrix[ord(amp[i]), ord(read[i + s])]) for i in range(max(0, -s), min(I, I - s)))


# ------------------------------------------------------------------------------------------------ running a batch
def counters(engine):
    pairs, singles = engine.path_counts()
    return dict(pairs=pairs, singles=singles, ring=engine.ring_counts(), diag=engine.diag_counts())


def run_switched(engine, refs, names, reads, matrix, go, ge, flags=0):
    """The batch with every shortcut as configured, then with C2B_NO_DIAG, C2B_NO_NARROW and F_NO_RING: records, alignments,
    aligned strings, edit lists and the count block must be identical.  -> counters of the default run"""
    buf, off = pack_reads(reads)
    out = []
    for env, fl in ((None, 0), ("C2B_NO_DIAG", 0), ("C2B_NO_NARROW", 0), (None, _lib.F_NO_RING)):
        if env:
            os.environ[env] = "1"
        try:
            engine.configure(refs, names, matrix, go, ge, 5, 2, flags | fl, ALPHA, 48)
            engine.counts_reset()
            res = engine.align_packed(buf, off)
            out.append((res, engine.counts_raw(), counters(engine)))
        finally:
            if env:
                os.environ.pop(env)
    a, ca, cnt = out[0]
    for b, cb, _ in out[1:]:
        assert (a.recs == b.recs).all() and (a.alns == b.alns).all() and (ca == cb).all()
        cols = np.arange(a.W)[None, :] >= (a.W - a.alns[:, 0]["aln_len"].astype(np.int64))[:, None]
        assert ((a.strings[:, 0] == b.strings[:, 0]) | ~cols[:, None, :]).all()
        (ea, fa), (eb, fb) = PU.edits_canonical(a), PU.edits_canonical(b)
        assert (fa == fb).all() and (ea[fa] == eb[fb]).all()
    assert out[1][2]["diag"][:2] == (0, 0) and out[3][2]["ring"] == (0, 0)
    return cnt


def check_point(engine, ref, matrix, go, ge, reads, oracle_reads=None):
    """run_switched + the oracle; -> (admission, counters)"""
    refs, names = {"Reference": ref}, ["Reference"]
    adm = admission(matrix, ref["sequence"], ref["gap_incentive"], go, ge)
    cnt = run_switched(engine, refs, names, reads, matrix, go, ge)
    P = O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge)
    PU.check_against_oracle(engine, refs, names, P, reads if oracle_reads is None else oracle_reads, matrix)
    return adm, cnt


def assert_paths(adm, cnt, reads, ref, matrix, go, ge):
    """the path counters agree with the restated admission (all reads no longer than pk_maxJ, or all longer)"""
    maxJ = max(len(r) for r in reads)
    if adm["pk_maxJ"] >= maxJ:
        assert cnt["singles"] == 0 and cnt["pairs"] > 0, cnt
    else:
        assert cnt["pairs"] == 0 and cnt["singles"] > 0, cnt
    # ring: (reads kept by the 72-slot band, reads sent on to the full matrix); diag[2]: reads the narrow tier sent to the
    # wide ring.  At 2 ge + gmax == smax the ring is admitted but its bound is at least smax * J: it runs and keeps nothing.
    if adm["rg_ok"] and adm["pk_maxJ"] >= maxJ and maxJ == len(ref["sequence"]):
        assert cnt["ring"][0] > 0 or cnt["diag"][2] > 0, cnt
    elif not adm["rg_ok"]:
        assert cnt["ring"][0] == 0 and cnt["diag"][2] == 0, cnt
    proved = DT.rule_count(reads, {"Reference": ref}, ["Reference"], go=go, ge=ge, matrix=matrix) if adm["dg_ok"] else 0
    assert cnt["diag"][0] == proved, (cnt, proved)
    if adm["dg_ok"]:
        assert cnt["diag"][0] + cnt["diag"][1] == len(reads), cnt
        assert proved > 0 or maxJ != len(ref["sequence"]), cnt
    else:
        assert cnt["diag"][:2] == (0, 0), cnt


def point_reads(rng, amp, cut, n, length=None):
    """amplicon-length reads with 0-3 substitutions (diagonal-tier candidates), reads with indels at the cut (ring), a few
    random ones, all cut or padded to `length` (default: the amplicon's; one length per batch keeps the tiers on)"""
    I = len(amp)
    reads = DT.edited_reads(rng, amp, [int(x) for x in rng.integers(0, 4, n // 2)])
    reads += [r.tobytes().decode() for r in synth.synth_reads(rng, amp, n - n // 2 - 2, I, sub_rate=0.01, del_frac=0.4,
                                                              ins_frac=0.3, cut=cut)]
    reads += ["".join(rng.choice(list("ACGT"), I)) for _ in range(2)]
    length = I if length is None else length
    return [(r + "".join(rng.choice(list("ACGT"), max(0, length - len(r)))))[:length] for r in reads]


# ------------------------------------------------------------------------------------------------ (b) predicate edges
def _gi(I, cut, value=1, **at):
    g = np.zeros(I + 1, dtype=np.int64)
    g[cut + 1] = value
    for k, v in at.items():
        g[int(k[1:])] = v
    return g


# name, matrix, go, ge, amplicon length, cut-site incentive, other incentive entries, read length, expected (pk on for the
# reads, rg_ok, dg_ok)
EDGES = [
    ("smin+2b=0", O.make_matrix(5, -4, -2, -1), -20, -2, 250, 1, {}, None, (True, True, True)),
    ("smin+2b=-1", O.make_matrix(5, -5, -2, -1), -20, -2, 250, 1, {}, None, (False, False, False)),
    ("smax+2b=1000", O.make_matrix(996, -4, -2, -1), -20, -2, 120, 1, {}, 6, (True, True, True)),
    ("smax+2b=1001", O.make_matrix(997, -4, -2, -1), -20, -2, 120, 1, {}, 6, (False, False, False)),
    ("gmax=64", asym(A_C=-3, G_T=-1), -20, -2, 40, 64, {}, None, (True, False, False)),
    ("gmax=65", asym(A_C=-3, G_T=-1), -20, -2, 40, 65, {}, None, (False, False, False)),
    ("2ge+gmax=smax", O.make_matrix(5, -4, -2, -1), -20, -2, 250, 9, {}, None, (True, True, False)),
    ("2ge+gmax=smax+1", O.make_matrix(5, -4, -2, -1), -20, -2, 250, 10, {}, None, (True, False, False)),
    ("2(ge+gp)=smax", O.make_matrix(6, -4, -2, -1), -20, -2, 250, 5, {}, None, (True, True, True)),
    ("2(ge+gp)=smax+1", O.make_matrix(5, -4, -2, -1), -20, -2, 250, 5, {}, None, (True, True, False)),
    ("gmin=0", asym(C_A=-3, T_G=-2), -12, -3, 200, 2, {"g0": 0, "g7": 0, "g200": 1}, None, (True, True, True)),
    ("gmin=-1", asym(C_A=-3, T_G=-2), -12, -3, 200, 2, {"g0": 0, "g7": -1, "g200": 1}, None, (False, False, False)),
    ("go==ge", O.make_matrix(4, -3, -1, 0), -4, -4, 250, 1, {"g0": 2}, None, (True, True, True)),
    ("go>ge", O.make_matrix(4, -3, -1, 0), -1, -5, 250, 1, {}, None, (False, False, False)),
    ("ge=0", O.make_matrix(6, -1, 0, 2), -6, 0, 250, 1, {}, None, (False, False, False)),
]


@pytest.mark.parametrize("edge", EDGES, ids=[e[0] for e in EDGES])
def test_admission_edges(eng, edge):
    engine, scale = eng
    name, m, go, ge, I, gcut, extra, length, (pk_on, rg_on, dg_on) = edge
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    amp = synth.random_amplicon(rng, I)
    ref = synth.amplicon_setup(amp, guide_start=I // 2 - 10, exclude_left=5, exclude_right=5)
    ref["gap_incentive"] = _gi(I, ref["cut_point"], gcut, **extra)
    adm = admission(m, amp, ref["gap_incentive"], go, ge)
    reads = point_reads(rng, amp, ref["cut_point"], 32 * scale, length)
    maxJ = max(len(r) for r in reads)
    assert (adm["pk_maxJ"] >= maxJ, adm["rg_ok"], adm["dg_ok"]) == (pk_on, rg_on, dg_on), adm
    _, cnt = check_point(engine, ref, m, go, ge, reads, reads[:24 * scale])
    assert_paths(adm, cnt, reads, ref, m, go, ge)
    for r in reads[:2] + reads[-3:-1]:                     # the single-call entry on the same scoring point
        assert align.global_align(r, amp, m, ref["gap_incentive"], go, ge, engine=engine) == \
            O.global_align(r, amp, m, ref["gap_incentive"], go, ge)


def test_packed_read_length_edge(eng):
    """smax + 2 beta = 40 puts pk_maxJ at 176 for a 250-bp amplicon: reads of 176 bp take the packed path, reads of 177 bp the
    32-bit path, in one-length batches and mixed in one batch."""
    engine, scale = eng
    m, go, ge = O.make_matrix(36, -4, -2, -1), -20, -2
    rng = np.random.default_rng(176)
    amp = synth.random_amplicon(rng, 250)
    ref = synth.amplicon_setup(amp)
    refs, names = {"Reference": ref}, ["Reference"]
    adm = admission(m, amp, ref["gap_incentive"], go, ge)
    K = adm["pk_maxJ"]
    assert K == 176, adm
    P = O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge)
    by_len = {}
    for J in (K, K + 1):
        by_len[J] = point_reads(rng, amp, ref["cut_point"], 16 * scale, J)
        engine.configure(refs, names, m, go, ge, 5, 2, 0, ALPHA, 48)
        engine.counts_reset()
        buf, off = pack_reads(by_len[J])
        engine.align_packed(buf, off)
        cnt = counters(engine)
        if J == K:
            assert cnt["singles"] == 0 and cnt["pairs"] > 0, cnt
        else:
            assert cnt["pairs"] == 0 and cnt["singles"] > 0, cnt
        PU.check_against_oracle(engine, refs, names, P, by_len[J], m)
    mixed = [r for pair in zip(by_len[K], by_len[K + 1]) for r in pair]
    PU.check_against_oracle(engine, refs, names, P, mixed, m)
    cnt = counters(engine)
    assert cnt["pairs"] > 0 and cnt["singles"] > 0, cnt
    for r in (by_len[K][0], by_len[K + 1][0]):
        assert align.global_align(r, amp, m, ref["gap_incentive"], go, ge, engine=engine) == \
            O.global_align(r, amp, m, ref["gap_incentive"], go, ge)


# ------------------------------------------------------------------------------------------------ (c) the diagonal bound
# A matrix whose A row holds five distinct scores, gap_extend -3 (so that the packed path admits smin = -5) and gap_open from
# -3 to -40: dg_S = 0, 1, 2, 3, 4.
TIE_M = asym(A_C=-3, A_G=-4, A_T=-5, A_N=-1)
TIE_GO = [-3, -4, -13, -22, -40]


def _tie_gi(rng, I):
    """non-zero gi[0] and gi[I], and gi[I - t] != gi[I - t + 1] for t = 1..4"""
    g = np.zeros(I + 1, dtype=np.int64)
    g[0], g[I] = int(rng.integers(1, 3)), int(rng.integers(1, 3))
    for t in range(1, 5):
        g[I - t] = (int(g[I - t + 1]) + 1 + int(rng.integers(0, 2))) % 3
    g[I // 2] = 2
    return g


def read_at_score(rng, m, amp, target, lo):
    """amp with substitutions / N at positions >= lo whose main-diagonal score is exactly `target` (None if not found)"""
    D0 = diag_score(m, amp, amp)
    for _ in range(300):
        s, rem = list(amp), D0 - target
        free = list(range(lo, len(amp)))
        rng.shuffle(free)
        for p in free:
            if rem == 0:
                break
            a = amp[p]
            opts = [b for b in ALPHA if b != a and 0 < int(m[ord(a), ord(a)] - m[ord(a), ord(b)]) <= rem]
            exact = [b for b in opts if int(m[ord(a), ord(a)] - m[ord(a), ord(b)]) == rem]
            if exact or opts:
                b = exact[0] if exact else opts[int(rng.integers(0, len(opts)))]
                s[p] = b
                rem -= int(m[ord(a), ord(a)] - m[ord(a), ord(b)])
        if rem == 0:
            return "".join(s)
    return None


@pytest.mark.parametrize("go", TIE_GO)
def test_diagonal_bound_straddling_reads(eng, go):
    """Reads whose diagonal score D equals dg_thr (left to the DP) and dg_thr + 1; on an all-A amplicon, reads whose D equals
    the exact score A(s) of offset diagonal s for every 1 <= |s| <= dg_S (ties: left to the DP), and A(s) + 1."""
    engine, scale = eng
    ge, m = -3, TIE_M
    rng = np.random.default_rng(-go)
    I = 80
    # random amplicon whose own seed test is one-sided: D == thr and D == thr + 1
    while True:
        amp = synth.random_amplicon(rng, I)
        ref = synth.amplicon_setup(amp, guide_start=30, exclude_left=5, exclude_right=5)
        if O._strand_choice(O.Params(), amp, ref) == "fw":
            break
    ref["gap_incentive"] = _tie_gi(rng, I)
    refs, names = {"Reference": ref}, ["Reference"]
    adm = admission(m, amp, ref["gap_incentive"], go, ge)
    assert adm["dg_ok"] and adm["S"] == TIE_GO.index(go), adm
    at, above = [], []
    while len(at) < 6 * scale or len(above) < 6 * scale:
        for lst, target in ((at, adm["thr"]), (above, adm["thr"] + 1)):
            r = read_at_score(rng, m, amp, target, 50)
            assert r is not None and diag_score(m, amp, r) == target
            lst.append(r)
    assert DT.rule_count(at, refs, names, go=go, ge=ge, matrix=m) == 0
    assert DT.rule_count(above, refs, names, go=go, ge=ge, matrix=m) > 0
    reads = at + above + [amp] * 4
    cnt = run_switched(engine, refs, names, reads, m, go, ge)
    assert cnt["diag"][0] == DT.rule_count(reads, refs, names, go=go, ge=ge, matrix=m)
    P = O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge)
    PU.check_against_oracle(engine, refs, names, P, reads, m)
    # all-A amplicon: D - A(s) is the score of the first s read bases (s > 0) or of the last |s| ones (s < 0) minus c(s)
    hom = "A" * I
    href = synth.amplicon_setup(hom, guide_start=30, exclude_left=5, exclude_right=5)
    href["gap_incentive"] = _tie_gi(rng, I)
    hrefs = {"Reference": href}
    adm = admission(m, hom, href["gap_incentive"], go, ge)
    assert adm["dg_ok"] and adm["S"] == TIE_GO.index(go), adm
    ties, near = [], []
    for s, cs in adm["c"].items():
        t = abs(s)
        for delta in (0, 1):
            combo = next((k for k in itertools.product(ALPHA, repeat=t) if sum(int(m[65, ord(b)]) for b in k) == cs + delta
                          and set(k) != {"A"}), None)
            if combo is None:
                continue
            r = "".join(combo) + hom[t:] if s > 0 else hom[:I - t] + "".join(combo)
            assert diag_score(m, hom, r) - diag_score(m, hom, r, s) == cs + delta
            (ties if delta == 0 else near).append(r)
    assert len(ties) >= len(adm["c"]) // 2
    assert DT.rule_count(ties, hrefs, names, go=go, ge=ge, matrix=m) == 0
    reads = (ties + near + [hom]) * 2
    reads = reads * max(1, (16 * scale + len(reads) - 1) // len(reads))
    cnt = run_switched(engine, hrefs, names, reads, m, go, ge)
    assert cnt["diag"][0] == DT.rule_count(reads, hrefs, names, go=go, ge=ge, matrix=m) > 0, cnt
    PU.check_against_oracle(engine, hrefs, names, P, ties + near + [hom], m)


# ------------------------------------------------------------------------------------------------ (d) narrow tier and ring
# name, matrix, go, ge, cut-site incentive, whether the narrow band's bound is ever beaten (the fixture's matrix scores matches
# 5..7, so a read's score stays far below the narrow bound 7 J - 163)
RING_POINTS = [
    ("make(4,-3,-1,0)", O.make_matrix(4, -3, -1, 0), -20, -2, 1, True),
    ("asym", asym(A_C=-3, C_A=-2, G_T=-4, T_G=-1, A_N=0), -12, -2, 2, True),
    ("file ge=-5", None, -5, -5, 3, False),
]


@pytest.mark.parametrize("point", RING_POINTS, ids=[p[0] for p in RING_POINTS])
def test_narrow_tier_and_ring_straddle_their_bounds(eng, point):
    """The read makers of the EDNAFULL checks (deletions, insertions, heavy substitution loads and random reads on both sides of
    ring_bound(.., 33, 31) and ring_bound(.., 17, 11)) under other matrices, gap pairs and incentives."""
    engine, scale = eng
    name, m, go, ge, gval, narrow_keeps = point
    if m is None:
        m = O.read_matrix(MATRIX_FILE)
    I = 250
    amp = synth.random_amplicon(np.random.default_rng(41), I)         # check_ring_equals_full's amplicon
    ref = synth.amplicon_setup(amp, guide_start=I // 2 - 10)
    gi = _gi(I, ref["cut_point"], gval, g0=1, g250=1)
    adm = admission(m, amp, gi, go, ge)
    assert adm["rg_ok"] and adm["pk_maxJ"] >= I, adm
    kept, sent = PU.check_ring_equals_full(engine, n=48 * scale, matrix=m, go=go, ge=ge, gap_incentive=gi, oracle_subset=24 * scale)
    assert kept > 0 and sent > 0
    amp = synth.random_amplicon(np.random.default_rng(59), I)         # check_narrow_equals_wide's amplicon
    ref = synth.amplicon_setup(amp, guide_start=I // 2 - 10)
    gi = _gi(I, ref["cut_point"], gval, g0=1, g250=1)
    adm = admission(m, amp, gi, go, ge)
    proved, tier1, tier2 = PU.check_narrow_equals_wide(engine, n=64 * scale, matrix=m, go=go, ge=ge, gap_incentive=gi,
                                                       oracle_subset=24 * scale)
    assert adm["dg_ok"] and tier2 > 0, (proved, tier1, tier2)          # the narrow tier ran and sent reads to the wide ring
    assert (tier1 > tier2) == narrow_keeps, (proved, tier1, tier2)


# ------------------------------------------------------------------------------------------------ (f) other paths
def test_hdr_three_amplicons_custom_matrix(eng):
    engine, scale = eng
    m = O.read_matrix(MATRIX_FILE)
    rng = np.random.default_rng(43)
    refs, names, reads = synth.hdr_workload(np.random.default_rng(42), rng, 48 * scale)
    reads = [bytes(r).decode() for r in reads]
    P = O.Params(needleman_wunsch_gap_open=-8, needleman_wunsch_gap_extend=-3, expected_hdr_amplicon_seq=refs[names[1]]["sequence"])
    PU.check_against_oracle(engine, refs, names, P, reads, m)


def test_pooled_ref_id_custom_matrix(eng):
    engine, scale = eng
    PU.check_pooled(engine, n_amplicons=4, reads_per=12 * scale, seed=23, matrix=asym(A_C=-3, C_A=-2, G_T=-4, T_G=-1, N_N=6),
                    go=-10, ge=-3)


# ------------------------------------------------------------------------------------------------ int32 headroom
def _defined(reads, amp, m, gi, go, ge):
    """the reads (and the reverse complements the seed test may add) on which the reference's traceback stays defined"""
    out = []
    for r in reads:
        try:
            for s in (r, O.reverse_complement(r)):
                O.global_align(s, amp, m, gi, go, ge)
            out.append(r)
        except O.OracleUndefined:
            pass
    return out


def test_large_scores_equal_the_reference_or_are_refused(eng):
    """EDNAFULL scaled by 2^16 .. 2^22 and by 3 * 2^17, incentives scaled up the same way: at every point the single call,
    the batch and the device-pointer entry either equal the oracle or refuse with C2B_E_LIMIT; never a different
    alignment.  Scales that fit (up to 3 * 2^17 for a 250-bp read and amplicon) must not be refused."""
    engine, scale = eng
    rng = np.random.default_rng(1)
    amp = synth.random_amplicon(rng, 250)
    ref = synth.amplicon_setup(amp)
    refs, names = {"Reference": ref}, ["Reference"]
    base = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 24 * scale, 250, sub_rate=0.02, cut=ref["cut_point"])]
    points = [(1 << k, 1) for k in range(16, 23)] + [(3 << 17, 1)] + [(1, 1 << k) for k in (10, 16, 20, 22, 27)] + [(1 << 16, 1 << 18)]
    refused = set()
    for ms, gs in points:
        m = O.make_matrix() * ms
        gi = np.asarray(ref["gap_incentive"], dtype=np.int64) * gs
        for r in base[:4]:
            try:
                want = O.global_align(r, amp, m, gi, -20, -2)
            except O.OracleUndefined:
                want = None                         # the reference's traceback reads a pointer it never set
            try:
                got = align.global_align(r, amp, m, gi, -20, -2, engine=engine)
            except EngineError as ex:
                assert "int32" in str(ex) or (want is None and "status" in str(ex)), ex
                if "int32" in str(ex):
                    refused.add((ms, gs))
                continue
            assert got == want, (ms, gs)
        rf = dict(ref, gap_incentive=gi)
        reads = _defined(base, amp, m, gi, -20, -2)
        if reads:
            try:
                PU.check_against_oracle(engine, {"Reference": rf}, names, O.Params(), reads, m)
                batch_refused = False
            except EngineError as ex:
                assert "int32" in str(ex), ex
                batch_refused = True
            assert batch_refused == ((ms, gs) in refused), (ms, gs)
        engine.configure({"Reference": rf}, names, m, -20, -2, 5, 2, 0, ALPHA, 48)
        rc = device_rc(engine, reads or base)
        assert rc == (_lib.E_LIMIT if (ms, gs) in refused else 0), (ms, gs, rc)
    assert (1 << 19, 1) in refused and (1 << 22, 1) in refused and (1, 1 << 27) in refused
    assert not refused & {(1 << 16, 1), (1 << 17, 1), (3 << 17, 1), (1, 1 << 10), (1, 1 << 16)}, refused


def test_gap_open_up_to_the_existing_guard(eng):
    """gap_open just inside |gap_open| * J * I < 2^28 equals the oracle; one step past it is refused."""
    engine, scale = eng
    rng = np.random.default_rng(3)
    amp = synth.random_amplicon(rng, 200)
    ref = synth.amplicon_setup(amp, guide_start=90)
    reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 16 * scale, 200, sub_rate=0.02, cut=ref["cut_point"])]
    go = -((1 << 28) // (200 * 200) - 1)
    reads = _defined(reads, amp, O.make_matrix(), ref["gap_incentive"], go, -2)
    assert len(reads) >= 8
    PU.check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(needleman_wunsch_gap_open=go), reads, O.make_matrix())
    assert align.global_align(reads[0], amp, O.make_matrix(), ref["gap_incentive"], go, -2, engine=engine) == \
        O.global_align(reads[0], amp, O.make_matrix(), ref["gap_incentive"], go, -2)
    with pytest.raises(EngineError):
        align.global_align(reads[0], amp, O.make_matrix(), ref["gap_incentive"], go - 2, -2, engine=engine)


def device_rc(engine, reads):
    """return code of one c2b_align_batch_device call over `reads` (outputs discarded)"""
    buf, off = pack_reads(reads)
    n, maxlen = len(reads), int(np.diff(off).max())
    W = engine.string_width(maxlen)
    host = [np.ascontiguousarray(buf), np.ascontiguousarray(off, dtype=np.int64)]
    outs = [np.zeros(n * 16, np.uint8), np.zeros(n * 32, np.uint8), np.zeros(n * 2 * W, np.uint8), np.zeros(n * 48 * 8, np.uint8)]
    if engine.lib_path is None or "emu" not in str(engine.lib_path):
        import torch
        keep = [torch.from_numpy(a).cuda() for a in host + outs]
        ptrs = [t.data_ptr() for t in keep]
    else:
        ptrs = [a.ctypes.data for a in host + outs]
    rc = engine.L.c2b_align_batch_device(engine.h, ptrs[0], ptrs[1], n, maxlen, None, None, None, ptrs[2], ptrs[3], ptrs[4], ptrs[5])
    if rc == 0:
        engine.sync()
    return rc
