"""Diagonal tier of the ALIGN kernel (c2b_diag_kernel): reads as long as their amplicon whose ungapped score beats every
other path are aligned on the main diagonal without a DP.  Every batch here runs twice, with the tier and with C2B_NO_DIAG=1
(the launch sequence without it), and the two runs must agree field by field: records, alignments, strings, edit lists, op
streams, compact outputs and the count block; subsets also go through the oracle.  The number of proved reads must equal a
numpy restatement of the rule (DESIGN.md section 3).  Runs on the CPU warp emulator; the same checks run through the sm_90a
library when a GPU is present."""
import os

import numpy as np
import pytest

import parity_util as PU
from crispresso2_b200 import _lib, synth
from crispresso2_b200.engine import Engine, pack_reads
from oracle import oracle as O

COMP = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}
ACGT = list("ACGT")


def rc(s):
    return "".join(COMP[c] for c in reversed(s))


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def emu(request):
    """the warp-emulator build; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0)
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build())


def device_batch(engine, reads, ref_id, cap=48):
    """One c2b_align_batch_device call (no pairing order: reads in their given order) -> (recs, alns, strings, edits) as
    bytes, every output buffer zero-filled first so that unwritten bytes compare equal."""
    buf, off = pack_reads(reads)
    n, maxlen = len(reads), int(np.diff(off).max())
    W = engine.string_width(maxlen)
    rid = np.ascontiguousarray(ref_id, dtype=np.int32)
    host = [np.ascontiguousarray(buf), np.ascontiguousarray(off, dtype=np.int64), rid]
    outs = [np.zeros(n * 16, np.uint8), np.zeros(n * 32, np.uint8), np.zeros(n * 2 * W, np.uint8), np.zeros(n * cap * 8, np.uint8)]
    if engine.lib_path is None or "emu" not in str(engine.lib_path):
        import torch
        dev = [torch.from_numpy(a).cuda() for a in host + outs]
        ptrs = [t.data_ptr() for t in dev]
        get = lambda: [t.cpu().numpy().tobytes() for t in dev[3:]]
    else:
        ptrs = [a.ctypes.data for a in host + outs]
        get = lambda: [a.tobytes() for a in outs]
    L = engine.L
    rc_ = L.c2b_align_batch_device(engine.h, ptrs[0], ptrs[1], n, maxlen, None, None, ptrs[2], ptrs[3], ptrs[4], ptrs[5], ptrs[6])
    assert rc_ == 0, L.c2b_last_error(engine.h)
    engine.sync()
    return get()


def run_both(engine, refs, names, reads, go=-20, ge=-2, flags=0, ref_id=None, matrix=None):
    """-> diag_counts of the default run; asserts that the run without the tier computed the same.  matrix: EDNAFULL if None."""
    m = O.make_matrix() if matrix is None else matrix
    buf, off = pack_reads(reads)
    n = len(reads)
    out = []
    for switch in (None, "1"):
        if switch:
            os.environ["C2B_NO_DIAG"] = switch
        try:
            engine.configure(refs, names, m, go, ge, 5, 2, flags, "ACGTN", 48)
            engine.counts_reset()
            res = engine.align_packed(buf, off, ref_id=ref_id)
            dc = engine.diag_counts()
            cres = engine.align_packed(buf, off, compact=True, ref_id=ref_id, count=np.zeros(n, dtype=np.int32),
                                       qweight=np.zeros(n, dtype=np.int32))
            out.append((res, engine.counts_raw(), cres, dc))
        finally:
            os.environ.pop("C2B_NO_DIAG", None)
    (a, ca, xa, da), (b, cb, xb, db) = out
    assert db[:2] == (0, 0), db                                   # C2B_NO_DIAG: the tier does not run
    assert (a.recs == b.recs).all() and (a.alns == b.alns).all() and (ca == cb).all()
    # columns and strand; the state byte names the kernel that aligned (a read the DP tiers take in another grouping may be
    # finished by the general kernel instead)
    assert ((xa.meta & 0xffffff) == (xb.meta & 0xffffff)).all() and (((xa.meta >> 24) != 0) == ((xb.meta >> 24) != 0)).all()
    cols = np.arange(a.W)[None, :] >= (a.W - a.alns[:, 0]["aln_len"].astype(np.int64))[:, None]     # right-aligned strings
    assert ((a.strings[:, 0] == b.strings[:, 0]) | ~cols[:, None, :]).all()
    (ea, fa), (eb, fb) = PU.edits_canonical(a), PU.edits_canonical(b)
    assert (fa == fb).all() and (ea[fa] == eb[fb]).all()
    nw = (xa.meta.reshape(-1) & 0xffff).astype(np.int64)
    ops_a, ops_b = xa.ops.reshape(len(nw), -1), xb.ops.reshape(len(nw), -1)
    for k in range(len(nw)):
        used = (int(nw[k]) + 31) // 32
        assert (ops_a[k, :used] == ops_b[k, :used]).all(), k
    return da


def rule_count(reads, refs, names, go=-20, ge=-2, ref_id=None, alphabet="ACGTN", matrix=None):
    """The proof rule restated on the host: reads of the amplicon's length, every base in the alphabet, one strand from the
    seed test, strictly above the bound on the other path classes and above the exact scores of the near offset diagonals."""
    m = O.make_matrix() if matrix is None else matrix
    params = O.Params()
    per_ref = []
    for name in names:
        ref = refs[name]
        seq = ref["sequence"]
        I = len(seq)
        gi = np.asarray(ref["gap_incentive"], dtype=np.int64)
        score_rows = np.array([[m[ord(seq[i]), ord(q)] for i in range(I)] for q in alphabet], dtype=np.int64)
        smax, gp, gmin = int(score_rows.max()), max(int(gi.max()), 0), int(gi.min())
        ok = go <= ge <= 0 and gmin >= 0 and 2 * (ge + gp) <= smax
        thr = max(smax * (I - 1) + go + ge + 2 * gp, go * I * I + max(smax, 0) * I + 2 * I * gp)
        edge = lambda t: smax * (I - t) + t * (2 * ge + gp) + gp
        S = 0
        while S < 4 and S + 1 < I and edge(S + 1) > thr:
            S += 1
        if S + 1 < I:
            thr = max(thr, edge(S + 1))
        c = {s: 2 * ge * abs(s) + int(gi[0]) + (int(gi[I - s]) if s > 0 else abs(s) * int(gi[I])) for s in range(-S, S + 1) if s}
        per_ref.append((ok, I, thr, S, c))
    total = 0
    for k, read in enumerate(reads):
        r = 0 if ref_id is None else int(ref_id[k])
        ok, I, thr, S, c = per_ref[r]
        ref = refs[names[r]]
        if not ok or len(read) != I or any(ch not in alphabet for ch in read):
            continue
        strand = O._strand_choice(params, read, ref)
        if strand == "both":
            continue
        s_read = read if strand == "fw" else rc(read)
        sub = lambda s: sum(int(m[ord(ref["sequence"][i]), ord(s_read[i + s])]) for i in range(max(0, -s), min(I, I - s)))
        d = sub(0)
        if d > thr and all(d > sub(s) + c[s] for s in c):
            total += 1
    return total


def edited_reads(rng, amp, n_subs_list, positions=None):
    out = []
    for k, ns in enumerate(n_subs_list):
        s = list(amp)
        pos = positions[k] if positions is not None else rng.choice(len(amp), ns, replace=False)
        for p in pos:
            s[p] = rng.choice([c for c in ACGT if c != amp[p]])
        out.append("".join(s))
    return out


def test_bench_like_batch(emu):
    """The bench's read mix (synth_reads_fast defaults: 0.5 %/base substitutions, 25 % deletions, 10 % insertions)."""
    rng = np.random.default_rng(5)
    amp = synth.random_amplicon(np.random.default_rng(42), 250)
    ref = synth.amplicon_setup(amp)
    n = 6144
    reads = [r.tobytes().decode() for r in synth.synth_reads_fast(rng, amp, n, 250, cut=ref["cut_point"])]
    refs, names = {"Reference": ref}, ["Reference"]
    proved, tier1, tier2 = run_both(emu, refs, names, reads)
    assert proved + tier1 == n
    assert proved == rule_count(reads, refs, names)
    frac = proved / n
    print("diagonal tier: %.1f %% of the bench-like reads proved" % (100 * frac))
    assert 0.5 < frac < 0.7, frac
    PU.check_against_oracle(emu, refs, names, O.Params(), reads[:400], O.make_matrix())


def test_substitutions_n_bases_and_reverse_complement(emu):
    rng = np.random.default_rng(11)
    amp = synth.random_amplicon(rng, 250)
    ref = synth.amplicon_setup(amp)
    cut = ref["cut_point"]
    reads = [amp] * 4
    for ns in range(1, 7):
        reads += edited_reads(rng, amp, [ns] * 6)
    I = len(amp)
    reads += edited_reads(rng, amp, [1] * 6, positions=[[0], [I - 1], [cut], [cut + 1], [0, I - 1], [cut - 1, cut + 2]])
    for p in (0, 7, cut, I - 1):
        reads.append(amp[:p] + "N" + amp[p + 1:])
    reads.append(amp[:30] + "NN" + amp[32:])
    reads += [rc(s) for s in reads[:40]]
    refs, names = {"Reference": ref}, ["Reference"]
    proved, tier1, _ = run_both(emu, refs, names, reads)
    assert proved == rule_count(reads, refs, names) and proved > 0 and tier1 > 0
    PU.check_against_oracle(emu, refs, names, O.Params(), reads, O.make_matrix())


def test_both_strand_and_other_lengths_go_to_the_dp(emu):
    rng = np.random.default_rng(12)
    while True:                                           # an amplicon whose own seed test is one-sided
        amp = synth.random_amplicon(rng, 250)
        ref = synth.amplicon_setup(amp)
        if O._strand_choice(O.Params(), amp, ref) == "fw":
            break
    both = [amp[:40] + "".join(rng.choice(ACGT, 170)) + amp[-40:] for _ in range(16)]       # few seeds: both strands
    short = [amp[:-1]] * 8 + [amp[1:]] * 8
    longer = [amp + "A"] * 16
    refs, names = {"Reference": ref}, ["Reference"]
    for reads in (both, short, longer):                   # one length per batch: no pairing order, the tiers run
        proved, tier1, _ = run_both(emu, refs, names, reads)
        assert proved == 0 and tier1 == len(reads)
    mixed = both[:8] + [amp] * 8 + both[8:]
    proved, _, _ = run_both(emu, refs, names, mixed)
    assert proved == 8 == rule_count(mixed, refs, names)
    PU.check_against_oracle(emu, refs, names, O.Params(), mixed, O.make_matrix())


@pytest.mark.parametrize("kind", ["tandem", "homopolymer"])
def test_repeats_where_a_shifted_diagonal_ties(emu, kind):
    """Amplicons whose shifted copy matches almost as well: a dinucleotide tandem repeat or homopolymer runs.  A tie between
    the main diagonal and an offset path must not be proved."""
    rng = np.random.default_rng(13 if kind == "tandem" else 14)
    if kind == "tandem":
        amp = "AC" * 125
    else:
        amp = "".join(c * 25 for c in ("A", "C", "G", "T", "A", "G", "C", "T", "A", "C"))
    ref = synth.amplicon_setup(amp, guide_start=100, seed_count=5)
    reads = [amp] * 4 + edited_reads(rng, amp, [1, 2, 3] * 8)
    reads += [amp[1:] + amp[-1], amp[-1] + amp[:-1], amp[2:] + amp[-2:], "A" + amp[:-1], amp[1:] + "C"]
    refs, names = {"Reference": ref}, ["Reference"]
    proved, _, _ = run_both(emu, refs, names, reads)
    assert proved == rule_count(reads, refs, names)
    PU.check_against_oracle(emu, refs, names, O.Params(), reads, O.make_matrix())


def test_tie_with_an_offset_diagonal_is_left_to_the_dp(emu):
    """A hand-made tie on an all-A amplicon: read C + A x 59 scores 59 x 5 - 4 = 291 on the main diagonal and 59 x 5 - 2 - 2
    = 291 on offset +1 (leading insertion, trailing deletion, no incentive there): not proved; the amplicon itself is."""
    amp = "A" * 60
    ref = synth.amplicon_setup(amp, guide_start=20, exclude_left=5, exclude_right=5)
    refs, names = {"Reference": ref}, ["Reference"]
    assert rule_count([amp], refs, names) == 1
    assert rule_count(["C" + amp[:-1]], refs, names) == 0
    reads = [amp] * 16 + ["C" + amp[:-1]] * 16
    proved, tier1, _ = run_both(emu, refs, names, reads)
    assert (proved, tier1) == (16, 16)
    PU.check_against_oracle(emu, refs, names, O.Params(), reads, O.make_matrix())


@pytest.mark.parametrize("go,ge,gi,expect_on", [(-20, -2, 1, True), (-10, -3, 2, True), (-5, -5, 0, True), (-20, -2, 5, False)])
def test_gap_settings(emu, go, ge, gi, expect_on):
    rng = np.random.default_rng(20 + gi)
    amp = synth.random_amplicon(rng, 200)
    ref = synth.amplicon_setup(amp, guide_start=80, gap_incentive_value=gi)
    reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 256, 200, sub_rate=0.01, cut=ref["cut_point"])]
    refs, names = {"Reference": ref}, ["Reference"]
    proved, tier1, _ = run_both(emu, refs, names, reads, go=go, ge=ge)
    assert (proved > 0) == expect_on and (tier1 > 0) == expect_on      # incentive 5 with gap_extend -2: the tier is off
    assert proved == (rule_count(reads, refs, names, go=go, ge=ge) if expect_on else 0)
    P = O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge)
    PU.check_against_oracle(emu, refs, names, P, reads[:96], O.make_matrix())


def test_pooled_ref_id_batch(emu):
    rng = np.random.default_rng(31)
    refs, names, reads, rid = {}, [], [], []
    for a in range(5):
        L = int(rng.integers(150, 260))
        amp = synth.random_amplicon(rng, L)
        name = "amp%d" % a
        refs[name] = synth.amplicon_setup(amp, guide_start=L // 2 - 10)
        names.append(name)
        rs = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 96, L, sub_rate=0.004, cut=refs[name]["cut_point"])]
        reads += rs
        rid += [a] * len(rs)
    order = rng.permutation(len(reads))
    reads = [reads[k] for k in order]
    ref_id = np.asarray(rid, dtype=np.int32)[order]
    # host batches of several amplicons get a pairing order (the narrow and diagonal tiers are off): the device-pointer API
    # takes the reads as given
    out = []
    for switch in (None, "1"):
        if switch:
            os.environ["C2B_NO_DIAG"] = switch
        try:
            emu.configure(refs, names, O.make_matrix(), -20, -2, 5, 2, 0, "ACGTN", 48)
            emu.counts_reset()
            out.append((device_batch(emu, reads, ref_id), emu.counts_raw(), emu.diag_counts()))
        finally:
            os.environ.pop("C2B_NO_DIAG", None)
    (a, ca, da), (b, cb, db) = out
    assert a == b and (ca == cb).all() and db[:2] == (0, 0)
    assert da[0] == rule_count(reads, refs, names, ref_id=ref_id) and da[0] > 0 and da[0] + da[1] == len(reads)


def test_hdr_three_amplicons_tier_off(emu):
    rng = np.random.default_rng(41)
    refs, names, reads = synth.hdr_workload(np.random.default_rng(42), rng, 512)
    reads = [bytes(r).decode() for r in reads]
    proved, tier1, _ = run_both(emu, refs, names, reads, flags=_lib.F_HDR_REF1)
    assert (proved, tier1) == (0, 0)
