"""Classification inside the diagonal tier: a read the tier proves (an ungapped alignment on the main diagonal) is classified
and counted by the tier itself, and CLASSIFY only visits the reads on the tier's list.  Every batch runs with the tier and
with C2B_NO_DIAG=1 (CLASSIFY over every read), through the host entry and the compact entry, and the two runs must agree:
records, alignments, strings, edit lists, op streams and the count block of each call -- which also checks the widest
alignment, since the compact copy-out sizes its strings and op words from it.  The cases are the decisions the tier now
makes: weights, min_aln_score, the ignore / discard / legacy flags, edit-list overflow, strings and edits switched off,
reverse-complement reads with N.  Runs on the CPU warp emulator; the same checks run on the sm_90a library with -m gpu."""
import os

import numpy as np
import pytest

import parity_util as PU
from crispresso2_b200 import _lib, synth
from crispresso2_b200.engine import Engine, pack_reads
from oracle import oracle as O
from test_diag_tier import edited_reads, rc, rule_count


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def eng(request):
    """the warp-emulator build; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0)
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build())


def amplicon(seed=3):
    amp = synth.random_amplicon(np.random.default_rng(seed), 250)
    return amp, synth.amplicon_setup(amp)


def mixed_reads(rng, amp, ref):
    """reads the tier proves (0-3 substitutions, N bases, both strands) mixed with indel reads it leaves to the DP tiers"""
    I = len(amp)
    reads = [amp] * 8 + edited_reads(rng, amp, [1] * 16 + [2] * 16 + [3] * 8)
    reads += edited_reads(rng, amp, [1] * 4, positions=[[0], [I - 1], [ref["cut_point"]], [0, I - 1]])
    for p in rng.choice(I, 8, replace=False):
        reads.append(amp[:p] + "N" + amp[p + 1:])
    reads.append(edited_reads(rng, amp, [1])[0][:40] + "N" + amp[41:])
    reads += [rc(s) for s in reads[:16] + reads[-9:]]                 # strand 1, N bases included
    reads += [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 48, I, sub_rate=0.004, cut=ref["cut_point"])]
    order = rng.permutation(len(reads))
    return [reads[k] for k in order]


def run_both(engine, refs, names, reads, flags=0, edit_cap=48, count=None, qweight=None, strings=True, edits=True):
    """-> diag_counts of the default run; asserts that the run without the tier computed the same through the host entry
    (with `strings`, `edits`) and through the compact entry (with `edits`)"""
    buf, off = pack_reads(reads)
    out = []
    for switch in (None, "1"):
        if switch:
            os.environ["C2B_NO_DIAG"] = switch
        try:
            engine.configure(refs, names, O.make_matrix(), -20, -2, 5, 2, flags, "ACGTN", edit_cap)
            engine.counts_reset()
            res = engine.align_packed(buf, off, count=count, qweight=qweight, strings=strings, edits=edits)
            dc = engine.diag_counts()
            cnt = engine.counts_raw()
            engine.counts_reset()
            cres = engine.align_packed(buf, off, count=count, qweight=qweight, edits=edits, compact=True)
            out.append((res, cnt, cres, engine.counts_raw(), dc))
        finally:
            os.environ.pop("C2B_NO_DIAG", None)
    (a, ca, xa, cxa, da), (b, cb, xb, cxb, db) = out
    assert db[:2] == (0, 0) and da[0] > 0, (da, db)
    assert (a.recs == b.recs).all() and (a.alns == b.alns).all() and (ca == cb).all()
    assert (xa.recs == xb.recs).all() and (xa.alns == xb.alns).all() and (cxa == cxb).all()
    assert (xa.recs == a.recs).all() and (xa.alns == a.alns).all()
    if strings:
        cols = np.arange(a.W)[None, :] >= (a.W - a.alns[:, 0]["aln_len"].astype(np.int64))[:, None]
        assert ((a.strings[:, 0] == b.strings[:, 0]) | ~cols[:, None, :]).all()
    if edits and edit_cap:
        for p, q in ((a, b), (xa, xb)):
            (ep, fp), (eq, fq) = PU.edits_canonical(p), PU.edits_canonical(q)
            assert (fp == fq).all() and (ep[fp] == eq[fq]).all()
    assert ((xa.meta & 0xffffff) == (xb.meta & 0xffffff)).all() and (((xa.meta >> 24) != 0) == ((xb.meta >> 24) != 0)).all()
    nw = (xa.meta.reshape(-1) & 0xffff).astype(np.int64)
    ops_a, ops_b = xa.ops.reshape(len(nw), -1), xb.ops.reshape(len(nw), -1)
    for k in range(len(nw)):
        used = (int(nw[k]) + 31) // 32
        assert (ops_a[k, :used] == ops_b[k, :used]).all(), k
    return da


def test_weights_and_counts(eng):
    """non-unit count and qweight (qweight 0: aligned but not counted)"""
    rng = np.random.default_rng(1)
    amp, ref = amplicon()
    reads = mixed_reads(rng, amp, ref)
    refs, names = {"Reference": ref}, ["Reference"]
    n = len(reads)
    count = rng.integers(1, 7, n).astype(np.int32)
    qweight = rng.integers(0, 4, n).astype(np.int32)
    proved, tier1, _ = run_both(eng, refs, names, reads, count=count, qweight=qweight)
    assert proved == rule_count(reads, refs, names) and proved + tier1 == n


@pytest.mark.parametrize("min_score", [99.5, 99.6, 100.0])
def test_min_aln_score_between_mismatch_counts(eng, min_score):
    """250 bp: 0, 1, 2 mismatches score 100.0, 99.6, 99.2; a proved read at or below min_aln_score is not aligned"""
    rng = np.random.default_rng(2)
    amp, ref = amplicon()
    ref = dict(ref, min_aln_score=min_score)
    reads = mixed_reads(rng, amp, ref)
    refs, names = {"Reference": ref}, ["Reference"]
    run_both(eng, refs, names, reads)
    a = eng.align(reads)
    aligned = a.recs["best_score_milli"] > 0
    assert aligned.any() != (min_score == 100.0) and not aligned.all()


@pytest.mark.parametrize("flags", [_lib.F_IGNORE_SUBSTITUTIONS, _lib.F_DISCARD_INDEL_READS, _lib.F_LEGACY_INS,
                                   _lib.F_DISCARD_INDEL_READS | _lib.F_LEGACY_INS | _lib.F_IGNORE_DELETIONS,
                                   _lib.F_EXPAND_AMBIGUOUS | _lib.F_ASSIGN_FIRST])
def test_flags(eng, flags):
    rng = np.random.default_rng(3)
    amp, ref = amplicon()
    reads = mixed_reads(rng, amp, ref)
    refs, names = {"Reference": ref}, ["Reference"]
    count = rng.integers(1, 4, len(reads)).astype(np.int32)
    run_both(eng, refs, names, reads, flags=flags, count=count)


@pytest.mark.parametrize("cap", [1, 2])
def test_edit_list_overflow(eng, cap):
    rng = np.random.default_rng(4)
    amp, ref = amplicon()
    reads = mixed_reads(rng, amp, ref)
    refs, names = {"Reference": ref}, ["Reference"]
    run_both(eng, refs, names, reads, edit_cap=cap)
    a = eng.align(reads)
    over = (a.alns[:, 0]["status"] & _lib.ST_EDIT_OVERFLOW) != 0
    assert over.any() and not over.all()


@pytest.mark.parametrize("strings,edits", [(False, True), (True, False), (False, False)])
def test_without_strings_or_edits(eng, strings, edits):
    rng = np.random.default_rng(5)
    amp, ref = amplicon()
    reads = mixed_reads(rng, amp, ref)
    run_both(eng, {"Reference": ref}, ["Reference"], reads, strings=strings, edits=edits)


def test_reverse_complement_reads_with_n(eng):
    """strand-1 reads with N bases and substitutions: the read string is the complement col_decode spells"""
    rng = np.random.default_rng(6)
    amp, ref = amplicon()
    I = len(amp)
    fw = []
    for p in rng.choice(I, 24, replace=False):
        s = edited_reads(rng, amp, [int(rng.integers(0, 3))])[0]
        fw.append(s[:p] + "N" + s[p + 1:])
    reads = [rc(s) for s in fw] + [rc(amp)] * 8
    refs, names = {"Reference": ref}, ["Reference"]
    proved, _, _ = run_both(eng, refs, names, reads, count=np.full(len(reads), 3, dtype=np.int32))
    assert proved == rule_count(reads, refs, names) and proved > len(reads) // 2
    a = eng.align(reads)
    assert (a.alns[:, 0]["strand"] == 1).all()
    PU.check_against_oracle(eng, refs, names, O.Params(), reads, O.make_matrix())


def test_all_reads_proved(eng):
    """a batch the tier proves entirely: CLASSIFY runs over an empty list, and the widest alignment comes from the tier alone"""
    rng = np.random.default_rng(7)
    amp, ref = amplicon()
    reads = [amp] * 16 + edited_reads(rng, amp, [1, 2] * 24)
    refs, names = {"Reference": ref}, ["Reference"]
    proved, tier1, _ = run_both(eng, refs, names, reads)
    assert (proved, tier1) == (len(reads), 0)
    PU.check_against_oracle(eng, refs, names, O.Params(), reads, O.make_matrix())
