"""The launch sequence of a batch (plan_batch, c2b_engine.cu): how many kernels each kind of batch launches.  The warp emulator
runs the kernels' own loops, one launch per step of the plan, so it counts what the sm_90a library counts; bench.py reports
that count per step.  Every batch runs twice, and the path, diagonal-tier and routing counters of the two runs must agree.
Runs on the CPU warp emulator; the same table is checked on the sm_90a library when a GPU is present."""
import os

import numpy as np
import pytest

from crispresso2_b200 import synth
from crispresso2_b200.engine import Engine
from oracle import oracle as O


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def engine(request):
    """the warp-emulator build; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0)
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build())


def _reads(rng, amp, n, length=250):
    return [r.tobytes().decode() for r in synth.synth_reads(rng, amp, n, length, sub_rate=0.01, cut=126)]


def _batch(case):
    """-> (refs, names, reads, ref_id, switch)"""
    rng = np.random.default_rng(5)
    amp = synth.random_amplicon(rng, 250)
    one = {"Reference": synth.amplicon_setup(amp)}
    if case in ("single", "no_route", "no_diag", "no_narrow", "no_split"):
        switch = {"single": None}.get(case, "C2B_" + case.upper())
        return one, ["Reference"], _reads(rng, amp, 64), None, switch
    if case == "few":
        return one, ["Reference"], _reads(rng, amp, 12), None, None
    if case == "hdr":
        refs, names, reads = synth.hdr_workload(rng, rng, 64)
        return refs, names, [r.tobytes().decode() for r in reads], None, None
    if case == "pooled":
        amp2 = synth.random_amplicon(rng, 250)
        refs = {"A": one["Reference"], "B": synth.amplicon_setup(amp2)}
        reads = [r for pair in zip(_reads(rng, amp, 32), _reads(rng, amp2, 32)) for r in pair]
        return refs, ["A", "B"], reads, np.tile(np.array([0, 1], dtype=np.int32), 32), None
    if case == "mixed":
        return one, ["Reference"], _reads(rng, amp, 32) + _reads(rng, amp, 32, 240), None, None
    assert case == "coding"
    ref = dict(one["Reference"], contains_coding_seq=True, exon_positions=list(range(40, 200)), splicing_positions=[],
               exon_len_mods=[0])
    return {"Reference": ref}, ["Reference"], _reads(rng, amp, 64), None, None


# launches per batch: the diagonal tier, ALIGN (narrow first tier or groups of eight), the second-tier ALIGN launch,
# CLASSIFY and the general kernel over the left-over pairs -- or the general kernel alone
LAUNCHES = [
    ("single", 5),          # one amplicon, >= 16 reads of one length, routing on
    ("no_route", 5),
    ("no_diag", 4),
    ("few", 4),             # fewer than 16 reads: no diagonal tier
    ("no_narrow", 3),       # no narrow tier, and with it no diagonal tier
    ("hdr", 3),             # three amplicons, every read against each: no narrow tier
    ("pooled", 3),          # ref_id with reads on two amplicons: a pairing order, no narrow tier
    ("mixed", 3),           # mixed read lengths: a pairing order
    ("no_split", 1),
    ("coding", 1),          # a coding sequence: the general kernel alone
]


@pytest.mark.parametrize("case,launches", LAUNCHES, ids=[c for c, _ in LAUNCHES])
def test_launches_per_batch(engine, case, launches):
    refs, names, reads, ref_id, switch = _batch(case)
    if switch:
        os.environ[switch] = "1"
    try:
        engine.configure(refs, names, O.make_matrix(), -20, -2, 5, 2, 0, "ACGTN", 48)
        runs = []
        for _ in range(2):
            engine.counts_reset()
            before = engine.launch_count()
            engine.align(reads, ref_id=ref_id)
            runs.append((engine.launch_count() - before, engine.path_counts(), engine.diag_counts(), engine.route_counts()))
    finally:
        if switch:
            os.environ.pop(switch, None)
    assert runs[0][0] == launches, runs
    assert runs[0] == runs[1], runs
