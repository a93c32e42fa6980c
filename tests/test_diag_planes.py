"""Popcount scoring in the diagonal tier: when every amplicon base has a code in A/C/G/T and the matrix over those codes is
two-valued (a match score, a mismatch score), a read of A/C/G/T only is scored from the match counts of its bit planes
instead of per-column profile gathers; every other read (any N, any other matrix) takes the gathers.  Both must give the
same proof, so every batch runs with and without the tier (test_diag_tier.run_both) and the outputs must agree field by
field; the proved count must equal the host restatement of the rule, and the number of reads the tier scored by popcounts
must be the number of eligible reads -- and 0 where the flag is off.  Runs on the CPU warp emulator; the same checks run
through the sm_90a library when a GPU is present."""
import os

import numpy as np
import pytest

import parity_util as PU
from crispresso2_b200 import synth
from crispresso2_b200.engine import Engine, pack_reads
from oracle import oracle as O
from test_diag_tier import edited_reads, rc, rule_count, run_both

ACGT = "ACGT"


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def emu(request):
    """the warp-emulator build; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0)
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build())


def offsets_scored(I, go, ge, gp=1, smax=5):
    """dg_S: the offset diagonals the tier scores exactly (c2b_configure)"""
    thr = max(smax * (I - 1) + go + ge + 2 * gp, go * I * I + max(smax, 0) * I + 2 * I * gp)
    S = 0
    while S < 4 and S + 1 < I and smax * (I - S - 1) + (S + 1) * (2 * ge + gp) + gp > thr:
        S += 1
    return S


def eligible(reads, ref, two=True):
    """reads the tier scores by popcounts: the amplicon's length, A/C/G/T only, one strand from the seed test"""
    if not two:
        return 0
    I, params = len(ref["sequence"]), O.Params()
    return sum(1 for r in reads if len(r) == I and set(r) <= set(ACGT) and O._strand_choice(params, r, ref) != "both")


def check(engine, amp, reads, go=-20, ge=-2, matrix=None, two=True, ref=None, oracle=48):
    """run_both, then the proved count against the rule and the popcount-scored count against `eligible`"""
    ref = ref or synth.amplicon_setup(amp, guide_start=max(0, len(amp) // 2 - 10))
    refs, names = {"Reference": ref}, ["Reference"]
    proved, tier1, _ = run_both(engine, refs, names, reads, go=go, ge=ge, matrix=matrix)
    assert proved + tier1 == len(reads)
    assert proved == rule_count(reads, refs, names, go=go, ge=ge, matrix=matrix)
    m = O.make_matrix() if matrix is None else matrix
    engine.configure(refs, names, m, go, ge, 5, 2, 0, "ACGTN", 48)
    engine.counts_reset()
    buf, off = pack_reads(reads)
    engine.align_packed(buf, off)
    assert engine.diag_counts()[0] == proved
    assert engine.diag_popcount_reads() == eligible(reads, ref, two)
    if oracle:
        P = O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge)
        PU.check_against_oracle(engine, refs, names, P, reads[:oracle], m)
    return proved


def boundary_reads(rng, amp):
    """the amplicon, one substitution in each of the first and last four columns and on both sides of every 32-column word
    boundary, pairs of them, and reads shifted by one and two columns"""
    I = len(amp)
    cols = sorted({*range(4), *range(I - 4, I), *[b + d for b in range(32, I, 32) for d in (-1, 0)]} & set(range(I)))
    reads = [amp] * 2 + edited_reads(rng, amp, [1] * len(cols), positions=[[p] for p in cols])
    reads += edited_reads(rng, amp, [2] * (len(cols) - 1), positions=[[a, b] for a, b in zip(cols, cols[1:])])
    reads += [amp[1:] + "A", "C" + amp[:-1], amp[2:] + "GT", "TG" + amp[:-2]]
    return reads


def test_bench_mix(emu):
    rng = np.random.default_rng(5)
    amp = synth.random_amplicon(np.random.default_rng(42), 250)
    ref = synth.amplicon_setup(amp)
    reads = [r.tobytes().decode() for r in synth.synth_reads_fast(rng, amp, 2048, 250, cut=ref["cut_point"])]
    assert check(emu, amp, reads, ref=ref, oracle=200) > 0


@pytest.mark.parametrize("go,ge,S", [(-5, -5, 0), (-10, -3, 1), (-16, -2, 2), (-20, -2, 3), (-30, -2, 4)])
def test_word_boundaries_at_each_offset_count(emu, go, ge, S):
    assert offsets_scored(250, go, ge) == S
    rng = np.random.default_rng(60 + S)
    amp = synth.random_amplicon(rng, 250)
    reads = boundary_reads(rng, amp)
    reads += [rc(r) for r in reads[:24]]
    check(emu, amp, reads, go=go, ge=ge)


@pytest.mark.parametrize("kind", ["tandem", "homopolymer"])
def test_repeats_score_the_offsets_exactly(emu, kind):
    """amplicons whose shifted copies nearly match: the offset diagonals' popcounts decide the proof"""
    amp = "AC" * 125 if kind == "tandem" else "".join(c * 25 for c in "ACGTAGCTAC")
    rng = np.random.default_rng(70)
    reads = [amp] * 4 + edited_reads(rng, amp, [1, 2, 3] * 8)
    reads += [amp[1:] + amp[-1], amp[-1] + amp[:-1], amp[2:] + amp[-2:], "A" + amp[:-1], amp[1:] + "C"]
    check(emu, amp, reads, ref=synth.amplicon_setup(amp, guide_start=100))


def test_reads_with_n_take_the_gathers(emu):
    rng = np.random.default_rng(80)
    amp = synth.random_amplicon(rng, 250)
    reads = boundary_reads(rng, amp)[:20]
    for p in (0, 31, 32, 125, 249):
        reads.append(amp[:p] + "N" + amp[p + 1:])
        reads.append(reads[p % 7][:p] + "N" + reads[p % 7][p + 1:])
    check(emu, amp, reads)


def test_amplicon_with_n_turns_the_popcounts_off(emu):
    rng = np.random.default_rng(90)
    amp = synth.random_amplicon(rng, 250)
    amp = amp[:200] + "N" + amp[201:]
    reads = [amp] * 4 + edited_reads(rng, amp, [1, 2] * 8) + [amp.replace("N", "A")] * 4
    check(emu, amp, reads, two=False)


def test_other_two_valued_matrix(emu):
    rng = np.random.default_rng(100)
    amp = synth.random_amplicon(rng, 250)
    m = O.make_matrix(match_score=4, mismatch_score=-3)
    reads = boundary_reads(rng, amp)
    check(emu, amp, reads, matrix=m)


def test_matrix_not_two_valued_turns_the_popcounts_off(emu):
    rng = np.random.default_rng(110)
    amp = synth.random_amplicon(rng, 250)
    m = O.make_matrix()
    m[ord("A"), ord("G")] = m[ord("G"), ord("A")] = -1            # one transition scored apart
    reads = boundary_reads(rng, amp)
    check(emu, amp, reads, matrix=m, two=False)


@pytest.mark.parametrize("L", [31, 32, 33, 250, 256])
def test_amplicon_lengths(emu, L):
    rng = np.random.default_rng(120 + L)
    amp = synth.random_amplicon(rng, L)
    ref = synth.amplicon_setup(amp, guide_start=max(0, L // 2 - 10), guide_len=min(20, L // 2), exclude_left=2,
                               exclude_right=2, min_aln_score=0)
    reads = boundary_reads(rng, amp)
    reads += [rc(r) for r in reads[:8]]
    check(emu, amp, reads, ref=ref)


@pytest.mark.parametrize("n", [17, 32 * 37 + 5])
def test_batch_sizes(emu, n):
    """a batch smaller than one unit of 32 reads, and one whose units do not fill the resident warps evenly"""
    rng = np.random.default_rng(130 + n)
    amp = synth.random_amplicon(rng, 250)
    ref = synth.amplicon_setup(amp)
    reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, n, 250, sub_rate=0.01, n_rate=0.002, cut=ref["cut_point"])]
    check(emu, amp, reads, ref=ref, oracle=32)
