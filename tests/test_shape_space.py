"""The engine against the oracle over the shape space: amplicon length I, read length J and the seed test (--aln_seed_len,
--aln_seed_count, --aln_seed_min), placed on both sides of every length edge of the device paths (DESIGN.md sections 3-6):

  row blocks of 256 (nrb) and a lane's 8 rows (kstar / lstar); 32-column words (route bit planes, CLASSIFY's column steps, op
  words per lane); strand_mode's 256-position scan blocks; the narrow band (RN_DLO / RN_DHI = 17 / 11) and the ring's RG_MAXD
  = 8; PK_MAX_ALN = 512 of the packed pair path, RG_COMBO and I + J <= 512 of the diagonal tier; dg_ok's I >= 2.

`shape_admission()` restates the length side of each path's rule in numpy.  It is not the proof: it says which path must
run, and the counters (path_counts, ring_counts, diag_counts, route_counts, band_reruns) must confirm it, so that a test meant
for a shortcut fails when only the fallback ran.  Every batch goes through the oracle, and again with every shortcut off
(C2B_NO_DIAG, C2B_NO_ROUTE, C2B_NO_NARROW, C2B_NO_SPLIT, F_NO_RING, F_NO_PAIRING): records, alignments, strings, edit lists
and the count block must be identical.

The seed lists here are the ones the reference itself builds (`reference_seeds`, CRISPRessoCORE.py:3210-3235), and the
seed-test settings go past the defaults 10 / 5 / 2 up to the build's limits (C2B_MAX_SEEDS tested seeds of at most
C2B_MAX_SEED_LEN bases), which must refuse loudly one step past them.

Runs on the CPU warp emulator; with -m gpu the same checks run through the sm_90a library with larger batches."""
import os
import sys

import numpy as np
import pytest

import parity_util as PU
import test_scoring_space as SS
from crispresso2_b200 import _lib, core, synth
from crispresso2_b200.engine import Engine, EngineError, pack_reads
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ACGT = list("ACGT")
COMP = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}
MAX_READ_LEN, MAX_ALN = 512, 1024                      # C2B_MAX_READ_LEN, C2B_MAX_ALN_LEN
PK_MAX_ALN, RG_COMBO, RG_MAXD = 512, 320, 8            # c2b_core.cuh
MAX_SEEDS, MAX_SEED_LEN = 8, 20                        # C2B_MAX_SEEDS, C2B_MAX_SEED_LEN
OFF_ENV = ("C2B_NO_DIAG", "C2B_NO_ROUTE", "C2B_NO_NARROW", "C2B_NO_SPLIT")
RING_KEEPS_FROM = 64      # amplicon length from which the ring keeps the batches' amplicon-like pairs (shorter: full matrix)


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def eng(request):
    """(engine, batch scale): the warp-emulator build with small batches; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0), 4
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build()), 1


def rc(s):
    return "".join(COMP[c] for c in reversed(s))


def rand_seq(rng, n):
    return "".join(rng.choice(ACGT, n)) if n > 0 else ""


# ------------------------------------------------------------------------------------------------ references
def reference_seeds(seq, seed_len, seed_count, exclude_left, exclude_right):
    """CRISPRessoCORE.py:3210-3235 restated: a seed every `seed_count` positions from exclude_left; a start whose k-mer occurs
    in the reverse complement or is already a seed moves right (the reset to position 0 tests the loop's start, not the moved
    one, as the reference does), at most 100 times; a seed whose reverse complement occurs in the amplicon is skipped."""
    L = len(seq)
    seq_rc = rc(seq)
    seeds, rc_seeds = [], []
    for seed_start in range(exclude_left, L - exclude_right - seed_len, seed_count):
        attempts = 0
        this = seed_start
        pot = seq[this:this + seed_len]
        while pot in seq_rc or pot in seeds:
            attempts += 1
            if attempts > 100:
                break
            if seed_start > L - seed_len:
                this = 0
            this += 1
            pot = seq[this:this + seed_len]
        seed_rc = rc(pot)
        if seed_rc in seq:
            continue
        if pot not in seq_rc:
            seeds.append(pot)
            rc_seeds.append(seed_rc)
    return seeds, rc_seeds


def shape_ref(seq, seed_len=10, seed_count=5, exclude=None, cut=None, window=1, min_aln_score=60):
    """refs[...] entry valid for any length >= 1 (synth.amplicon_setup indexes past the end below ~25 bp): cut point inside the
    amplicon, excluded ends no wider than a quarter of it, seeds by the reference's rule."""
    I = len(seq)
    cut = max(0, min(I - 1, I // 2 - 1)) if cut is None else cut
    ex = min(15, I // 4) if exclude is None else exclude
    gi = np.zeros(I + 1, dtype=np.int64)
    gi[cut + 1] = 1
    win = set(range(cut - window + 1, cut + window + 1)) & set(range(ex, I - ex))
    fw, rv = reference_seeds(seq, seed_len, seed_count, ex, ex)
    return {"sequence": seq, "sequence_length": I, "gap_incentive": gi, "include_idxs": np.array(sorted(win), dtype=np.int64),
            "fw_seeds": fw, "rc_seeds": rv, "min_aln_score": min_aln_score, "cut_point": cut}


def shape_reads(rng, amp, J, n):
    """n reads of exactly J bases drawn from the amplicon: the amplicon itself, substitutions only, N bases, deletions of 8 / 9 /
    16 / 17 and insertions of 9 / 10 / 11 / 12 bases (either side of the narrow band's 17 / 11 and of the ring's 8), reverse
    complements and random reads; cut or padded with random bases to J."""
    I = len(amp)
    out = []
    for k in range(n):
        kind = k % 10
        mid = int(rng.integers(0, I + 1))
        if kind == 0:
            s = amp
        elif kind == 1:
            s = list(amp)
            for p in rng.choice(I, min(I, int(rng.integers(1, 4))), replace=False):
                s[p] = rng.choice([c for c in ACGT if c != s[p]])
            s = "".join(s)
        elif kind == 2:
            s = list(amp)
            for p in rng.choice(I, min(I, int(rng.integers(1, 3))), replace=False):
                s[p] = "N"
            s = "".join(s)
        elif kind in (3, 4):
            d = (8, 9, 16, 17)[k // 10 % 4]
            a = int(rng.integers(0, max(1, I - d + 1)))
            s = amp[:a] + amp[a + d:]
        elif kind in (5, 6):
            s = amp[:mid] + rand_seq(rng, (9, 10, 11, 12)[k // 10 % 4]) + amp[mid:]
        elif kind == 7:
            s = rc(amp)
        elif kind == 8:
            s = rc(amp[:mid] + rand_seq(rng, 1) + amp[mid:])
        else:
            s = rand_seq(rng, J)
        out.append((s + rand_seq(rng, max(0, J - len(s))))[:J])
    return out


# ------------------------------------------------------------------------------------------------ the host's rules, restated
def shape_admission(I, J, n, matrix=None, gi=None, go=-20, ge=-2, seq=None):
    """The length side of each path's rule for a batch of n reads of one length J against one amplicon of length I (the
    scoring side comes from test_scoring_space.admission):
      pair     the packed 16-bit pair path of the general kernel: J <= pk_maxJ, I + J <= PK_MAX_ALN
      align    the ALIGN kernel's packed groups of four pairs: J <= pk_maxJ, J <= RG_COMBO
      ring     the 72-slot ring of those groups: rg_ok (one row block, I <= 256), |J - I| <= RG_MAXD, I + J <= PK_MAX_ALN
      diag     the diagonal tier is launched (16 reads or more) over an admitted amplicon (dg_ok: I >= 2)
      prove    it may prove reads: J == I, J <= RG_COMBO, J <= pk_maxJ, I + J <= PK_MAX_ALN
      route    its routing test (rt_ok: I <= 256) may send reads straight to the wide ring
    everything else: the general kernel, one read per warp over the full matrix (32-bit)."""
    m = O.make_matrix() if matrix is None else matrix
    if gi is None:
        gi = np.zeros(I + 1, dtype=np.int64)
        gi[max(0, min(I - 1, I // 2 - 1)) + 1] = 1
    adm = SS.admission(m, "A" * I if seq is None else seq, gi, go, ge)
    pk = J <= adm["pk_maxJ"]
    ring = adm["rg_ok"] and pk and J <= RG_COMBO and I + J <= PK_MAX_ALN and abs(J - I) <= RG_MAXD
    diag = adm["dg_ok"] and n >= 16
    return dict(adm, pair=pk and I + J <= PK_MAX_ALN, align=pk and J <= RG_COMBO, ring=ring, diag=diag,
                prove=diag and J == I and J <= RG_COMBO and pk and I + J <= PK_MAX_ALN, route=diag and I <= 256)


def proved_count(reads, ref, params, matrix=None, go=-20, ge=-2):
    """the diagonal tier's proof rule (DESIGN.md section 3) with the seed test's settings of `params`"""
    m = O.make_matrix() if matrix is None else matrix
    seq = ref["sequence"]
    I = len(seq)
    gi = np.asarray(ref["gap_incentive"], dtype=np.int64)
    adm = SS.admission(m, seq, gi, go, ge)
    if not adm["dg_ok"]:
        return 0
    total = 0
    for read in reads:
        if len(read) != I or I + len(read) > PK_MAX_ALN or len(read) > RG_COMBO or len(read) > adm["pk_maxJ"]:
            continue
        strand = O._strand_choice(params, read, ref)
        if strand == "both":
            continue
        s = read if strand == "fw" else rc(read)
        d = SS.diag_score(m, seq, s)
        if d > adm["thr"] and all(d > SS.diag_score(m, seq, s, k) + c for k, c in adm["c"].items()):
            total += 1
    return total


# ------------------------------------------------------------------------------------------------ running a batch
def counters(engine):
    pairs, singles = engine.path_counts()                  # first: the other counters are read with it
    return dict(pairs=pairs, singles=singles, ring=engine.ring_counts(), diag=engine.diag_counts(), route=engine.route_counts(),
                reruns=engine.band_reruns())


def _run(engine, refs, names, reads, params, matrix, env=(), flags=0):
    for k in env:
        os.environ[k] = "1"
    try:
        engine.configure(refs, names, matrix, params.needleman_wunsch_gap_open, params.needleman_wunsch_gap_extend,
                         params.aln_seed_count, params.aln_seed_min, flags, "ACGTN", 48)
        engine.counts_reset()
        buf, off = pack_reads(reads)
        res = engine.align_packed(buf, off)
        return res, engine.counts_raw(), counters(engine)
    finally:
        for k in env:
            os.environ.pop(k, None)


def same_results(a, ca, b, cb):
    """records, alignments, aligned strings, edit lists and the count block of two runs of one batch"""
    assert (a.recs == b.recs).all() and (a.alns == b.alns).all() and (ca == cb).all()
    for r in range(a.alns.shape[1]):
        cols = np.arange(a.W)[None, :] >= (a.W - a.alns[:, r]["aln_len"].astype(np.int64))[:, None]
        assert ((a.strings[:, r] == b.strings[:, r]) | ~cols[:, None, :]).all()
        (ea, fa), (eb, fb) = PU.edits_canonical(a, r), PU.edits_canonical(b, r)
        assert (fa == fb).all() and (ea[fa] == eb[fb]).all()


def run_shape(engine, ref, reads, params=None, matrix=None, oracle=True):
    """One batch of one amplicon: shortcuts as configured, with C2B_NO_DIAG + C2B_NO_NARROW (every read through the ALIGN
    kernel's groups, where the ring's admission shows), and with every shortcut off; all three must compute the same, and the
    counters must show the paths shape_admission says.  -> (admission, counters of the default run)"""
    P = O.Params() if params is None else params
    m = O.make_matrix() if matrix is None else matrix
    go, ge = P.needleman_wunsch_gap_open, P.needleman_wunsch_gap_extend
    refs, names = {"Reference": ref}, ["Reference"]
    a, ca, cnt = _run(engine, refs, names, reads, P, m)
    b, cb, cgrp = _run(engine, refs, names, reads, P, m, env=("C2B_NO_DIAG", "C2B_NO_NARROW"))
    c, cc, cgen = _run(engine, refs, names, reads, P, m, env=("C2B_NO_SPLIT",))
    d, cd, coff = _run(engine, refs, names, reads, P, m, env=OFF_ENV, flags=_lib.F_NO_RING | _lib.F_NO_PAIRING)
    for x, cx in ((b, cb), (c, cc), (d, cd)):
        same_results(a, ca, x, cx)
    n = len(reads)
    assert coff["pairs"] == 0 and coff["ring"] == (0, 0) and coff["diag"] == (0, 0, 0) and coff["route"] == (0, 0), coff
    assert cgrp["diag"] == (0, 0, 0) and cgrp["route"] == (0, 0), cgrp
    assert cgen["diag"] == (0, 0, 0) and cgen["route"] == (0, 0), cgen
    lens = {len(r) for r in reads}
    if len(lens) != 1:
        if oracle:
            PU.check_against_oracle(engine, refs, names, P, reads, m)
        return None, dict(cnt, grp=cgrp, gen=cgen)
    J, I = lens.pop(), len(ref["sequence"])
    adm = shape_admission(I, J, n, m, ref["gap_incentive"], go, ge, ref["sequence"])
    why = (I, J, adm["pair"], adm["align"], adm["ring"], adm["diag"], adm["prove"])
    # the general kernel: a work item of two reads takes the packed pair path iff the lengths admit it, else two 32-bit reads
    items = (n + 1) // 2
    assert (cgen["pairs"], cgen["singles"]) == ((items, 0) if adm["pair"] else (0, items)), (why, cgen)
    # the ALIGN kernel's groups: every full group of four pairs is taken when the packed DP admits the length; the ring keeps
    # pairs only when the band can hold the alignment, the rest of the group's pairs take the full matrix
    if adm["align"]:
        assert sum(cgrp["ring"]) >= 4 * (n // 8), (why, cgrp)
    else:
        assert cgrp["ring"] == (0, 0), (why, cgrp)
    one_sided = sum(1 for r in reads if O._strand_choice(P, r, ref) != "both")
    if adm["ring"] and I >= RING_KEEPS_FROM and 4 * one_sided >= 3 * n:
        assert cgrp["ring"][0] > 0 and cgen["ring"][0] > 0, (why, cgrp, cgen)
    if not adm["ring"]:
        assert cgrp["ring"][0] == 0 and cgen["ring"][0] == 0 and cnt["ring"][0] == 0 and cnt["diag"][2] == 0, (why, cgrp, cnt)
    # the diagonal tier lists every read when it runs and proves exactly the reads the restated rule proves; its routing
    # test looks only at reads of the amplicon's length
    if adm["diag"]:
        assert cnt["diag"][0] + cnt["diag"][1] == n and sum(cnt["route"]) == cnt["diag"][1], (why, cnt)
        want = proved_count(reads, ref, P, m, go, ge) if adm["prove"] else 0
        assert cnt["diag"][0] == want, (why, cnt, want)
        if not adm["prove"]:
            assert cnt["route"][0] == 0, (why, cnt)
    else:
        assert cnt["diag"][:2] == (0, 0) and cnt["route"] == (0, 0), (why, cnt)
    if oracle:
        PU.check_against_oracle(engine, refs, names, P, reads, m)
    return adm, dict(cnt, grp=cgrp, gen=cgen)


def plant(rng, base, at, forbid, params, ref, want):
    """`base` with the seeds `at` = [(position, seed)] written in, every other occurrence of a seed in `forbid` broken by a
    substitution outside the planted windows, until the oracle's seed test gives `want` ('fw' / 'rc' / 'both')"""
    s = list(base)
    for p, k in at:
        s[p:p + len(k)] = list(k)
    keep = set()
    for p, k in at:
        keep.update(range(p, p + len(k)))
    for _ in range(200):
        t = "".join(s)
        hit = next(((t.find(k, 0), k) for k in forbid if k and k in t and not set(range(t.find(k), t.find(k) + len(k))) <= keep), None)
        if hit is None:
            break
        free = [q for q in range(hit[0], hit[0] + len(hit[1])) if q not in keep]
        q = free[int(rng.integers(0, len(free)))]
        s[q] = rng.choice([c for c in ACGT if c != s[q]])
    t = "".join(s)
    assert O._strand_choice(params, t, ref) == want, (t, at)
    return t


def strand_traps(rng, ref, J, params, edges):
    """Reads of J bases whose better strand is the reverse complement but whose seed test says 'fw' (exactly seed_min + 1
    forward seeds, one of them at each position in `edges`, no reverse seed) or 'both' (seed_min forward seeds): a seed
    test that miscounts by one changes the strand the oracle aligns, and so the result."""
    amp = ref["sequence"]
    ns = min(params.aln_seed_count, len(ref["fw_seeds"]))
    fw, rv = ref["fw_seeds"][:ns], ref["rc_seeds"][:ns]
    base = (rc(amp) + rand_seq(rng, J))[:J]
    out = []
    for e in edges:
        for extra, want in ((1, "fw"), (0, "both")):
            k = params.aln_seed_min + extra
            if not 1 <= k <= ns or e + len(fw[0]) > J:
                continue
            others = [x for x in range(0, J - len(fw[0]) + 1, len(fw[0]) + 1) if abs(x - e) > len(fw[0])]
            if len(others) < k - 1:
                continue
            pos = [e] + [others[i] for i in rng.choice(len(others), k - 1, replace=False)]
            out.append(plant(rng, base, list(zip(pos, fw[:k])), fw[k:] + rv, params, ref, want))
    return out


# ------------------------------------------------------------------------------------------------ (2) lengths
AMP_LENGTHS = [1, 2, 3, 7, 8, 9, 16, 17, 18, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 512, 513, 767, 768, 769]


def read_lengths(I, seed_len=10):
    """J in {1, 2, 3}, seed_len - 1 and seed_len, I - 9, I - 8, I, I + 8, I + 9 and 512 - I - 1 .. 512 - I + 1, inside the build's
    limits (1 <= J <= 512, I + J <= 1024)"""
    js = {1, 2, 3, seed_len - 1, seed_len, I - 9, I - 8, I, I + 8, I + 9, 511 - I, 512 - I, 513 - I}
    return sorted(j for j in js if 1 <= j <= MAX_READ_LEN and I + j <= MAX_ALN)


@pytest.mark.parametrize("I", AMP_LENGTHS)
def test_length_sweep(eng, I):
    """Every read length of read_lengths(I) against an amplicon of I bases, one length per batch (so that the tiers run):
    at least 32 reads plus an odd one at J == I (a full diagonal unit, two narrow units and a tail), 16 elsewhere.  Amplicons
    under 64 bp get seeds short enough to survive the reference's rule on them (length I // 3, one every base, none excluded,
    --aln_seed_min 0), so that their reads can pass the seed test and reach the diagonal tier."""
    engine, scale = eng
    rng = np.random.default_rng(1000 + I)
    amp = rand_seq(rng, I)
    if I >= 64:
        L, P, ref = 10, O.Params(), shape_ref(amp)
    else:
        L = max(1, min(10, I // 3))
        P = O.Params(aln_seed_count=1, aln_seed_min=0)
        ref = shape_ref(amp, seed_len=L, seed_count=1, exclude=0)
    seen = {}
    for J in read_lengths(I, L):
        n = (32 * scale + 1) if J == I else 16 * scale
        seen[J] = run_shape(engine, ref, shape_reads(rng, amp, J, n), params=P)
    if 2 <= I <= 256 and ref["fw_seeds"]:               # the diagonal tier proved amplicon-length reads
        assert seen[I][1]["diag"][0] > 0, seen[I]
    if I == 1:                                         # dg_ok needs I >= 2: the tier never runs
        assert not seen[1][0]["diag"] and seen[1][1]["diag"][:2] == (0, 0)


@pytest.mark.parametrize("I,J", [(2, 1), (1, 2), (512, 512), (511, 512), (512, 1), (1, 512)])
def test_alignment_width_edges(eng, I, J):
    """Alignments of 1 column up to I + J = 1024 columns, on both sides of the 512 columns of the single-word op streams."""
    engine, scale = eng
    rng = np.random.default_rng(7 * I + J)
    amp = rand_seq(rng, I)
    run_shape(engine, shape_ref(amp), shape_reads(rng, amp, J, 8 * scale))


def test_alignment_widths_around_32_columns(eng):
    """Mixed-length batches whose widest alignment sits just below, on and just above a multiple of 32 columns (the compact
    outputs' width Wt and CLASSIFY's column steps)."""
    engine, scale = eng
    rng = np.random.default_rng(32)
    for I, top in ((20, 12), (20, 13), (40, 24), (40, 25), (100, 92), (100, 93), (150, 170), (150, 171)):
        amp = rand_seq(rng, I)
        reads = [r for J in (max(1, top - 5), top) for r in shape_reads(rng, amp, J, 4 * scale)]
        reads += [amp[:top]] if top <= I else [amp + rand_seq(rng, top - I)]
        run_shape(engine, shape_ref(amp), reads)


@pytest.mark.parametrize("J", [255, 256, 257, 263, 264, 265, 511, 512])
def test_seed_in_the_second_scan_block(eng, J):
    """strand_mode scans 256 start positions per block: reads of 255-512 bases against a 280-bp amplicon whose third forward
    seed starts at position 256 or ends exactly at J, built so that missing that seed turns 'fw' into 'both' (or 'both' into
    'rc') and the better strand is the reverse complement."""
    engine, scale = eng
    rng = np.random.default_rng(J)
    amp = rand_seq(rng, 280)
    ref = shape_ref(amp)
    P = O.Params()
    edges = [J - 10] + ([256] if 256 + 10 <= J else []) + [0]
    traps = strand_traps(rng, ref, J, P, edges)
    assert len(traps) >= 4
    reads = (traps * (8 * scale // len(traps) + 1))[:8 * scale] + shape_reads(rng, amp, J, 8 * scale)
    run_shape(engine, ref, reads)


# ------------------------------------------------------------------------------------------------ (3) the seed test
SEED_LENS, SEED_COUNTS = (1, 2, 9, 19, 20), (1, 2, 7, 8)


def seed_mins(count):
    return (-1, 0, count - 1, count)


def seed_reads(rng, ref, P, J):
    """reads of the amplicon's length for one seed setting: shape_reads, a tested seed at position 0 and at J - L, a forward /
    reverse-complement chimera (hits on both strands), N inside a seed window, and the strand traps"""
    amp = ref["sequence"]
    I = len(amp)
    reads = shape_reads(rng, amp, J, 20)
    fw = ref["fw_seeds"][:max(0, min(P.aln_seed_count, len(ref["fw_seeds"])))]
    for k in fw[:2]:
        reads.append((k + amp[len(k):])[:J])
        reads.append((amp[:J - len(k)] + k)[-J:] if J >= len(k) else amp[:J])
    reads.append((amp[:I // 2] + rc(amp)[I // 2:])[:J])
    for k in fw[:2]:
        p = amp.find(k)
        if p >= 0:
            reads.append(amp[:p + len(k) // 2] + "N" + amp[p + len(k) // 2 + 1:])
    if fw:
        reads += strand_traps(rng, ref, J, P, [0, J - len(fw[0])])
    return reads


@pytest.mark.parametrize("L", SEED_LENS)
@pytest.mark.parametrize("count", SEED_COUNTS)
def test_seed_settings(eng, L, count):
    """--aln_seed_len L and --aln_seed_count count, with two of the seed_min values -1, 0, count - 1, count; seeds by the
    reference's rule over a 150-bp amplicon (a 1-bp seed never survives it); one-length batches with the counters checked,
    then reads shorter than L and of other lengths through the oracle."""
    engine, scale = eng
    rng = np.random.default_rng(100 * L + count)
    amp = rand_seq(rng, 150)
    ref = shape_ref(amp, seed_len=L, seed_count=count)
    assert all(len(k) == L for k in ref["fw_seeds"]) and len(ref["fw_seeds"]) == len(ref["rc_seeds"])
    if L == 1:
        assert ref["fw_seeds"] == []
    mins = seed_mins(count)
    for smin in (mins[(L + count) % 4], mins[(L + count + 2) % 4]):
        P = O.Params(aln_seed_count=count, aln_seed_min=smin)
        reads = seed_reads(rng, ref, P, 150)
        reads = (reads * (32 * scale // len(reads) + 1))[:32 * scale + 1]
        run_shape(engine, ref, reads, params=P)
        short = [amp[:max(1, L - 1)], amp[10:10 + L], rc(amp)[:L], amp[:75] + rc(amp)[:75], amp[:140], amp + "ACGTACGT"]
        run_shape(engine, ref, short + reads[:16], params=P)


def no_seed_hits(rng, ref, read):
    """`read` with one substitution inside every occurrence of a forward or reverse seed: no hit on either strand"""
    s = list(read)
    for k in ref["fw_seeds"] + ref["rc_seeds"]:
        while k in "".join(s):
            p = "".join(s).find(k) + len(k) // 2
            s[p] = rng.choice([c for c in ACGT if c != s[p]])
    return "".join(s)


@pytest.mark.parametrize("seeded", [False, True])
def test_negative_seed_min_reverse_complement_merge(eng, seeded):
    """Regression: under --aln_seed_min -1 a read with no seed hit on either strand passes the seed test as forward-only, and
    so does its reverse complement, so the read can align while its reverse complement does not.  The reference merges a
    read with its reverse complement only when both are in variantCache (CRISPRessoCORE.py:3964-3975); the count block used
    to take the merged weight regardless, and its class counts and vectors differed from the reference's.  Amplicons without
    seeds, and amplicons with seeds where the read has every seed broken; the read before and after its reverse complement."""
    engine, scale = eng
    rng = np.random.default_rng(101 + seeded)
    amp = rand_seq(rng, 150)
    ref = shape_ref(amp, seed_len=10 if seeded else 1, seed_count=5 if seeded else 1)
    assert bool(ref["fw_seeds"]) == seeded
    P = O.Params(aln_seed_count=5 if seeded else 1, aln_seed_min=-1)
    zero = [no_seed_hits(rng, ref, r) for r in shape_reads(rng, amp, 150, 10)]
    assert all(O._strand_choice(P, r, ref) == "fw" == O._strand_choice(P, rc(r), ref) for r in zero)
    reads = []
    for k, r in enumerate(zero):
        reads += [r, rc(r)] * (1 + k % 2) if k % 3 else [rc(r), r, r]
    reads += shape_reads(rng, amp, 150, 8 * scale)
    cache_o = O.process_reads(reads, {"Reference": ref}, ["Reference"], P, O.make_matrix())[0]
    assert any(r in cache_o and rc(r) not in cache_o for r in zero)      # the case that used to go wrong
    PU.check_against_oracle(engine, {"Reference": ref}, ["Reference"], P, reads, O.make_matrix())


def test_amplicons_without_seeds(eng):
    """Amplicons shorter than exclude_left + exclude_right + seed_len, and a reverse-complement-symmetric one (every k-mer is
    in its reverse complement): no seed, every read both-strand, and the amplicon itself ties on the two strands (the reverse
    complement is taken only when strictly better, CRISPRessoCORE.py:678-687)."""
    engine, scale = eng
    rng = np.random.default_rng(77)
    half = rand_seq(rng, 60)
    sym = half + rc(half)
    for amp, ex in ((rand_seq(rng, 34), 12), (rand_seq(rng, 30), 10), (sym, 15)):
        ref = shape_ref(amp, exclude=ex)
        assert ref["fw_seeds"] == [] and ref["rc_seeds"] == []
        reads = shape_reads(rng, amp, len(amp), 32 * scale)
        adm, cnt = run_shape(engine, ref, reads)
        assert cnt["diag"][0] == 0, cnt
        if adm["diag"]:
            assert cnt["diag"][2] == len(reads), cnt
    assert O._strand_choice(O.Params(), sym, shape_ref(sym)) == "both" and O.global_align(sym, sym, O.make_matrix(),
        shape_ref(sym)["gap_incentive"], -20, -2)[2] == O.global_align(rc(sym), sym, O.make_matrix(), shape_ref(sym)["gap_incentive"], -20, -2)[2]


@pytest.mark.parametrize("count", [1, 5, 8])
def test_all_both_strand_batch(eng, count):
    """seed_min >= count: no read can pass the seed test, so every read is aligned on both strands.  The diagonal tier proves
    none, the narrow tier keeps none (every read goes straight to the wide ring), and every read equals the oracle."""
    engine, scale = eng
    rng = np.random.default_rng(300 + count)
    amp = rand_seq(rng, 200)
    ref = shape_ref(amp, seed_count=count)
    P = O.Params(aln_seed_count=count, aln_seed_min=count)
    reads = shape_reads(rng, amp, 200, 48 * scale) + [amp, rc(amp)] * 8
    assert all(O._strand_choice(P, r, ref) == "both" for r in reads)
    adm, cnt = run_shape(engine, ref, reads, params=P)
    assert adm["diag"] and cnt["diag"] == (0, len(reads), len(reads)), cnt
    assert cnt["route"] == (len(reads), 0), cnt                  # both-strand reads skip the narrow tier


def test_hdr_three_amplicons_seed_tests_disagree(eng):
    """HDR mode with three amplicons under --aln_seed_len 19 --aln_seed_count 7 --aln_seed_min 0: the seed tests of one read
    disagree across the amplicons (forward for some, both strands for others), ref1 vectors included."""
    engine, scale = eng
    rng = np.random.default_rng(19)
    amp = rand_seq(rng, 220)
    hdr = amp[:100] + "TGA" + amp[103:107] + "ACGTAC" + amp[107:]
    third = amp[:20] + rand_seq(rng, 140) + amp[160:]
    seqs = {"WT": amp, "HDR": hdr, "OTHER": third}
    refs = {k: shape_ref(s, seed_len=19, seed_count=7, cut=105) for k, s in seqs.items()}
    names = ["WT", "HDR", "OTHER"]
    P = O.Params(aln_seed_count=7, aln_seed_min=0, expected_hdr_amplicon_seq=hdr)
    reads = []
    for s in (amp, hdr, third):
        reads += shape_reads(rng, s, 220, 16 * scale)
    reads += [amp[:110] + rc(hdr)[110:], third[:80] + rc(amp)[80:]]
    modes = [tuple(O._strand_choice(P, r, refs[n]) for n in names) for r in reads]
    assert sum(1 for m in modes if len(set(m)) > 1) >= 4
    PU.check_against_oracle(engine, refs, names, P, reads, O.make_matrix())


# ------------------------------------------------------------------------------------------------ the seed limits
def _fastq(tmp_path, reads):
    fq = tmp_path / "r.fastq"
    with open(fq, "w") as fh:
        for k, s in enumerate(reads):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))
    return str(fq)


def test_seed_limits_refused_before_any_launch(eng, tmp_path):
    """C2B_MAX_SEEDS = 8 tested seeds and seeds of C2B_MAX_SEED_LEN = 20 bases run and equal the oracle; 9 tested seeds or
    21-base seeds are refused with C2B_E_LIMIT by configure and, as EngineError, by process_fastq -- before any launch."""
    engine, scale = eng
    rng = np.random.default_rng(21)
    amp = rand_seq(rng, 200)
    reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 16 * scale, 200, sub_rate=0.01, rc_frac=0.3, cut=99)]
    m = O.make_matrix()
    for L, count, ok in ((10, MAX_SEEDS, True), (10, MAX_SEEDS + 1, False), (MAX_SEED_LEN, 5, True), (MAX_SEED_LEN + 1, 5, False)):
        ref = shape_ref(amp, seed_len=L, seed_count=count)
        assert len(ref["fw_seeds"]) > MAX_SEEDS and {len(k) for k in ref["fw_seeds"]} == {L}
        refs, names = {"Reference": ref}, ["Reference"]
        P = O.Params(aln_seed_count=count, aln_seed_min=0)
        if ok:
            engine.configure(refs, names, m, -20, -2, count, 0, 0, "ACGTN", 48)
            PU.check_against_oracle(engine, refs, names, P, reads, m)
            continue
        before = engine.launch_count()
        with pytest.raises(EngineError) as ex:
            engine.configure(refs, names, m, -20, -2, count, 0, 0, "ACGTN", 48)
        assert "(%d)" % _lib.E_LIMIT in str(ex.value) and ("C2B_MAX_SEEDS" in str(ex.value) or "seed length" in str(ex.value))
        args = PU.args_from({k: getattr(P, k) for k in vars(P)})
        with pytest.raises(EngineError):
            core.process_fastq(_fastq(tmp_path, reads), {}, names, refs, args, [], str(tmp_path), engine=engine, aln_matrix=m)
        assert engine.launch_count() == before
    # fewer seeds than the count: only the seeds that exist are tested, so a large count over a short amplicon still runs
    ref = shape_ref(amp[:60], seed_len=10, seed_count=20)
    assert len(ref["fw_seeds"]) <= MAX_SEEDS
    P = O.Params(aln_seed_count=20, aln_seed_min=0)
    PU.check_against_oracle(engine, {"Reference": ref}, ["Reference"], P, [r[:60] for r in reads], m)


# ------------------------------------------------------------------------------------------------ (4) annotations, CLI
def _annotation_env(tmp):
    import annotate_util as AU
    if not AU.have_reference():
        pytest.skip("needs oracle/_ref/install (built by __graft_entry__.build())")
    return AU


def test_annotation_pass_at_width_edges(eng, tmp_path):
    """--fastq_output / --bam_output annotations (op word l on lane l of the annotation kernel) against the reference's own
    process_fastq_write_out / process_single_fastq_write_bam_out, with inputs captured from its main(): alignments of 1 to about 63
    columns on a 32-bp amplicon ('-' strand reads included), and of 500 to about 1000 columns on a 500-bp amplicon (every op
    word lane in use), insertions in the first and last column."""
    engine, scale = eng
    AU = _annotation_env(tmp_path)
    sys.path.insert(0, os.path.join(os.path.dirname(HERE)))
    from baseline import ref_shim
    old_path = os.environ["PATH"]
    os.environ["PATH"] = AU.fake_samtools(str(tmp_path / "bin"))
    try:
        rng = np.random.default_rng(512)
        core_mod = ref_shim.load_core()
        for I in (32, 500):
            amp = rand_seq(rng, I)
            guide = amp[6:26] if I == 32 else amp[200:220]
            reads = [amp, rc(amp), amp[:1], amp[:2], "A" + amp, amp + "T", amp[:I // 2] + "G" + amp[I // 2:], rc(amp[1:]),
                     amp[:I - 1], amp + rand_seq(rng, min(MAX_READ_LEN, 31 if I == 32 else 12) - 0)]
            if I == 500:
                reads += [amp[:250] + rand_seq(rng, 13) + amp[250:499], rand_seq(rng, 500), rand_seq(rng, 480) + amp[-20:],
                          amp[:12] + rand_seq(rng, 488), rc(amp)[:400], amp[250:] + rand_seq(rng, 262),
                          rand_seq(rng, 262) + amp[:250]]
            reads = [r[:MAX_READ_LEN] for r in reads]
            fq = AU.write_fastq(str(tmp_path / ("w%d.fastq" % I)), reads)
            ex = ["--exclude_bp_from_left", "0", "--exclude_bp_from_right", "0"] if I == 32 else []
            ref_names, refs, args = AU.capture(tmp_path, ["-r1", fq, "-a", amp, "-g", guide] + ex)
            d = tmp_path / ("p%d" % I)
            d.mkdir()
            P = AU.Pair(core_mod, engine, d, ref_names, refs, args)
            res_r, res_b, cache_r, cache_b, text_r, text_b, untouched = P.fastq(fq, "f")
            assert untouched and text_r == text_b and text_r.count(b"\n") >= 4
            AU.check_results(res_r, res_b, cache_r, cache_b)
            res_r, res_b, cache_r, cache_b, sam_r, sam_b = P.sam(fq, "s")
            assert sam_r == sam_b
            AU.check_results(res_r, res_b, cache_r, cache_b)
            key = "variant_" + ref_names[0]
            strands = {v[key]["aln_strand"] for v in cache_r.values() if key in v}
            assert "-" in strands and "+" in strands, strands
    finally:
        os.environ["PATH"] = old_path


def test_cli_seed_settings_byte_identical(tmp_path):
    """The launcher against the unmodified reference CLI with --aln_seed_len 20 --aln_seed_count 8 --aln_seed_min 0: the seed
    lists come from the reference's own main(), and every output file is byte-identical."""
    import test_cli_dropin as CD
    if not CD.HAVE_REF:
        pytest.skip("needs oracle/_ref/install (built by __graft_entry__.build())")
    import build_emu
    lib = build_emu.build()
    import pe_case
    fq = os.path.join(str(tmp_path), "FANC.Cas9.fastq")
    with open(fq, "w") as fh:
        fh.write(pe_case.fanc_fastq_text())
    fanc, _ = __import__("annotate_util").amplicons()
    argv = ["-r1", fq, "-a", fanc, "-g", "GGAATCCCTTCTGCAGCACC", "--aln_seed_len", "20", "--aln_seed_count", "8",
            "--aln_seed_min", "0"]
    ref_dir, b200_dir = str(tmp_path / "ref"), str(tmp_path / "b200")
    CD._run("reference", "default", ref_dir, argv)
    rep = CD._run("b200", lib, b200_dir, argv)
    a, b = CD._snapshot(ref_dir), CD._snapshot(b200_dir)
    assert sorted(a) == sorted(b)
    assert not [k for k in a if a[k] != b[k]]
    assert len(a) >= 10 and CD._info_stats(ref_dir) == CD._info_stats(b200_dir)
    assert rep["checked"] > 20 and not rep["mismatch"], rep["mismatch"]
