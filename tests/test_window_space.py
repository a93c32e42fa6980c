"""The engine against the oracle over the quantification window, refs[name]['include_idxs']: the set of amplicon positions
whose edits count as "in the window" (DESIGN.md section 1).  It decides substitution_n / insertion_n / deletion_n and so
MODIFIED / UNMODIFIED, --discard_indel_reads and the ignore flags, the INS / DEL / SUB and length vectors, the size
histograms, N_MODS_IN_WINDOW / N_MODS_OUTSIDE_WINDOW / N_SUBS_OUTSIDE_WINDOW, the --coding_seq frameshift and splicing
block, the annotation pass's DEL= / INS= / SUB= fields and the allele tables' n_deleted / n_inserted / n_mutated.

The window is read in five separately written places: the host (c2b_configure builds the `incl` bit and the `cum` / `cumx`
/ `cums` prefix counts, dropping values outside [0, I)), CLASSIFY (column space: deletion runs by prefix count, insertions
on both flanks or either under legacy, flank de-duplication), the diagonal tier (substitutions only), the general kernel
(row space, also behind c2b_classify_aligned) and the annotation pass (the edit list's in_window bit).  The reference
builds windows of several runs (a union of per-guide windows, -qwc), windows touching position 0 or I - 1, the whole
amplicon (-w 0 / no guide, minus the excluded ends) and empty windows (-qwc 0, a cloned amplicon whose window mapping
lands nowhere).  `window_shapes()` gives each of these for one amplicon length, and `edge_reads()` plants edits on every
run boundary: a window whose run boundaries disagree with the edits' positions by one, or a run test that looks only at a
deletion's ends, changes the result.  `coverage()` proves from the oracle's own payloads that every boundary saw an
in-window and an out-of-window substitution, insertion and deletion, so the suite cannot drift into testing only one side.

Runs on the CPU warp emulator; with -m gpu the same checks run through the sm_90a library with larger batches."""
import os
import sys

import numpy as np
import pytest

import golden_util as G
import parity_util as PU
import test_reference_space as RS
import test_shape_space as SH
from crispresso2_b200 import core, resources, synth
from crispresso2_b200.engine import Engine
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ACGT = list("ACGT")
rc = SH.rc
AMP_LENGTHS = [40, 250, 300]          # 40: short; 250: diagonal tier, narrow and wide ring; 300: two row blocks, no ring
IGNORE = ("ignore_substitutions", "ignore_insertions", "ignore_deletions")
FLAG_SETS = [("plain", {}), ("legacy", {"use_legacy_insertion_quantification": True}),
             ("discard_indel", {"discard_indel_reads": True})] + [(f, {f: True}) for f in IGNORE]


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def eng(request):
    """(engine, on_gpu): the warp-emulator build with small batches; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0), True
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build()), False


# ------------------------------------------------------------------------------------------------ windows
def window_shapes(I):
    """name -> sorted list of inclusive runs (lo, hi) for an amplicon of I bases"""
    m = I // 2
    s = {"one_run": [(m - I // 8, m + I // 8)],                                       # the control: what every other suite uses
         "two_runs_hole1": [(m - 9, m - 1), (m + 1, m + 6)],
         "two_runs_hole2": [(m - 9, m - 2), (m + 1, m + 6)],
         "singletons": [(m - 6, m - 6), (m - 4, m - 4), (m - 1, m - 1), (m + 3, m + 3)],
         "from_zero": [(0, m)],
         "to_end": [(m, I - 1)],
         "both_ends": [(0, 4), (I - 5, I - 1)],
         "whole": [(0, I - 1)],
         "minus15": [(15, I - 16)],                                                   # what -w 0 gives
         "empty": []}
    if I >= 128:
        b = m - 50                                                  # holes of 1, 2 and 33: the wide one crosses a 32-column step
        s["four_runs"] = [(b, b + 10), (b + 12, b + 20), (b + 23, b + 30), (b + 64, b + 80)]
        s["at32"] = [(32, 63), (64, 64), (66, 95), (97, 128)]       # run edges on multiples of 32 and next to them
    else:
        s["four_runs"] = [(2, 8), (10, 15), (18, 22), (26, 36)]
    return s


def runs_of(idx):
    """the inclusive runs of a sorted position list"""
    out = []
    for p in idx:
        if out and p == out[-1][1] + 1:
            out[-1] = (out[-1][0], p)
        else:
            out.append((p, p))
    return out


def window_ref(seq, runs, cut=None, extra=(), min_aln_score=60, **kw):
    """SH.shape_ref with include_idxs = the positions of `runs` plus `extra` (values the engine must ignore)"""
    ref = SH.shape_ref(seq, cut=cut, min_aln_score=min_aln_score, **kw)
    idx = sorted({p for lo, hi in runs for p in range(lo, hi + 1)})
    ref["include_idxs"] = np.array(idx + list(extra), dtype=np.int64)
    return ref


def boundaries(runs, I):
    """every run's lo - 1, lo, hi, hi + 1 inside [0, I)"""
    return sorted({b for lo, hi in runs for b in (lo - 1, lo, hi, hi + 1) if 0 <= b < I})


# ------------------------------------------------------------------------------------------------ reads
def other(rng, *avoid):
    return rng.choice([c for c in ACGT if c not in avoid])


def amplicon(rng, I):
    """a random amplicon without two equal neighbours: every 1-bp deletion has one place, so an edit planted next to a
    window edge stays there"""
    s = [rng.choice(ACGT)]
    while len(s) < I:
        s.append(other(rng, s[-1]))
    return "".join(s)


def insert_at(rng, amp, p, k):
    """amp with k bases inserted between positions p - 1 and p; the inserted bases differ from both neighbours, so the
    aligner has no equal-scoring place to shift the gap to"""
    return amp[:p] + "".join(other(rng, amp[p - 1], amp[p]) for _ in range(k)) + amp[p:]


def delete(amp, a, b):
    """amp without positions [a, b), or None when the run could shift (amp[a] == amp[b] or amp[a - 1] == amp[b - 1])"""
    I = len(amp)
    if not 0 <= a < b <= I or (b < I and amp[a] == amp[b]) or (a > 0 and amp[a - 1] == amp[b - 1]):
        return None
    return amp[:a] + amp[b:]


def edge_reads(rng, amp, runs):
    """Edits planted on every run boundary b (lo - 1, lo, hi, hi + 1): a substitution and an N at b, insertions of 1 and 3
    bases with flanks (b - 1, b) and (b, b + 1), deletions that start at b and end at b, deletions that cover exactly one
    hole, that span a hole from one run into the next and that cover one whole run (ends out, middle in), deletions at the
    first and last columns, reads whose only edits lie outside the window, reads with two substitutions on window edges
    (proved by the diagonal tier at amplicon length), and reverse complements of some of them."""
    I = len(amp)
    win = {p for lo, hi in runs for p in range(lo, hi + 1)}
    bs = boundaries(runs, I) or boundaries([(I // 2 - 5, I // 2 + 5)], I)
    out = [amp]
    for b in bs:
        out.append(amp[:b] + other(rng, amp[b]) + amp[b + 1:])
        out.append(amp[:b] + "N" + amp[b + 1:])
        for k in (1, 3):
            if 1 <= b:
                out.append(insert_at(rng, amp, b, k))
            if b + 1 <= I - 1:
                out.append(insert_at(rng, amp, b + 1, k))
        for d in range(1, 9):
            r = delete(amp, b, b + d)
            if r:
                out.append(r)
                break
        for d in range(1, 9):
            r = delete(amp, b - d + 1, b + 1)
            if r:
                out.append(r)
                break
    for (lo0, hi0), (lo1, hi1) in zip(runs, runs[1:]):
        out += [r for r in (delete(amp, hi0 + 1, lo1), delete(amp, hi0, lo1 + 1), delete(amp, hi0 - 1, lo1 + 2)) if r]
    for lo, hi in runs:
        if hi - lo < 24:
            out += [r for r in (delete(amp, lo - d, hi + 1 + d) for d in (1, 2, 3, 4)) if r][:2]
    out += [r for r in (amp[1:], amp[2:], amp[:1] + amp[2:], amp[:1] + amp[3:], amp[:-1], amp[:-2], amp[:-2] + amp[-1:]) if r]
    outside = [p for p in range(2, I - 2) if not win & set(range(p - 1, p + 2))]
    for p in outside[::max(1, len(outside) // 4)][:4]:
        out.append(amp[:p] + other(rng, amp[p]) + amp[p + 1:])
        out.append(insert_at(rng, amp, p, 2))
        r = delete(amp, p, p + 1)
        if r:
            out.append(r)
    edges = [b for lo, hi in runs for b in (lo, hi + 1) if 0 <= b < I] or [I // 2]
    for j, b in enumerate(edges):                                   # two substitutions on window edges
        c = edges[(j + 1) % len(edges)]
        s = list(amp)
        s[b] = other(rng, amp[b])
        if c != b:
            s[c] = other(rng, amp[c])
        out.append("".join(s))
    out += [rc(s) for s in out[1::5]]
    return out


# ------------------------------------------------------------------------------------------------ coverage
def coverage(reads, ref, params=None):
    """From the oracle's payloads: for every run edge (inside position q, outside neighbour q'), which of 'sub_in' / 'sub_out',
    'ins_in' / 'ins_out', 'del_in' / 'del_out' occur.  An in-window edit touches q (an insertion: with both flanks in the
    window); an out-of-window one touches q' and reaches up to the edge.  -> {(q, q'): set of tags}"""
    P = O.Params() if params is None else params
    I = len(ref["sequence"])
    cache, _, _ = O.process_reads(reads, {"R": ref}, ["R"], P, O.make_matrix())
    runs = runs_of(sorted(int(v) for v in ref["include_idxs"] if 0 <= v < I))
    edges = [(lo, lo - 1) for lo, hi in runs] + [(hi, hi + 1) for lo, hi in runs]
    seen = {e: set() for e in edges}
    for v in cache.values():
        p = v["variant_R"]
        sub_in, sub_all = set(p["substitution_positions"]), set(p["all_substitution_positions"])
        ins_in = set(map(tuple, p["insertion_coordinates"]))
        flat = p["all_insertion_positions"]
        ins_all = {(flat[k], flat[k + 1]) for k in range(0, len(flat), 2)}
        del_in = set(map(tuple, p["deletion_coordinates"]))
        del_all = set(map(tuple, p["all_deletion_coordinates"]))
        for (q, q2), tags in seen.items():
            lo_side = q2 < q
            if q in sub_in:
                tags.add("sub_in")
            if q2 in sub_all - sub_in:
                tags.add("sub_out")
            if any(q in c for c in ins_in):
                tags.add("ins_in")
            if any(set(c) == {q, q2} for c in ins_all - ins_in):
                tags.add("ins_out")
            if any(a <= q < b and (a == q if lo_side else b == q + 1) for a, b in del_in):
                tags.add("del_in")
            if any(a <= q2 < b and (b == q if lo_side else a == q + 1) for a, b in del_all - del_in):
                tags.add("del_out")
    return seen


def check_coverage(reads, ref, I):
    """every run edge has its in-window and (where the neighbour exists) out-of-window substitution, insertion and deletion;
    an in-window insertion needs two window positions, so runs of one position have none"""
    runs = runs_of(sorted(int(v) for v in ref["include_idxs"] if 0 <= v < I))
    for (q, q2), tags in coverage(reads, ref).items():
        run = next(r for r in runs if r[0] <= q <= r[1])
        want = {"sub_in", "del_in"} | ({"ins_in"} if run[1] > run[0] and 1 <= q <= I - 2 else set())
        if 0 <= q2 < I:
            want |= {"sub_out", "ins_out"}
        if 4 <= q2 < I - 4:              # closer to an end the aligner trades a deletion for an end gap and mismatches
            want.add("del_out")
        assert want <= tags, ((q, q2), sorted(want - tags))


# ------------------------------------------------------------------------------------------------ (1) shapes x edges x flags
SHAPE_CASES = [(I, name) for I in AMP_LENGTHS for name in window_shapes(I)]


@pytest.mark.parametrize("I,shape", SHAPE_CASES)
def test_window_shape(eng, I, shape):
    """One window shape over an amplicon of I bases, reads planted on every run boundary: the batch with every shortcut on,
    with C2B_NO_DIAG + C2B_NO_NARROW, with C2B_NO_SPLIT and with every shortcut off must compute the same, and equal the
    oracle (SH.run_shape); then the same reads under --use_legacy_insertion_quantification, --discard_indel_reads and each
    ignore flag against the oracle (the emulator runs two of these five per case, rotating, so every flag meets every
    amplicon length; the GPU runs all five).  Coverage of every edge is checked from the oracle's payloads; at 250 bp the diagonal
    tier must have proved reads."""
    engine, gpu = eng
    rng = np.random.default_rng(I * 100 + sorted(window_shapes(I)).index(shape))
    amp = amplicon(rng, I)
    runs = window_shapes(I)[shape]
    ref = window_ref(amp, runs, min_aln_score=40 if I < 64 else 60)
    reads = edge_reads(rng, amp, runs)
    if runs:
        check_coverage(reads, ref, I)
    if gpu:
        reads = reads * 4 + SH.shape_reads(rng, amp, I, 256)
    # reads of the amplicon's length in a batch of their own (the narrow and diagonal tiers take one-length batches only)
    same = [r for r in reads if len(r) == I]
    if len(same) < 16:                                               # one diagonal unit at least
        same = (same + [rc(r) for r in same]) * 2
    assert len(same) >= 16
    adm, cnt = SH.run_shape(engine, ref, same)
    if I == 250:
        assert adm["prove"] and cnt["diag"][0] > 0, cnt
    SH.run_shape(engine, ref, reads)
    k = SHAPE_CASES.index((I, shape))
    for name, kw in FLAG_SETS[1:] if gpu else [FLAG_SETS[1 + k % 5], FLAG_SETS[1 + (k + 2) % 5]]:
        PU.check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(**kw), reads, O.make_matrix())


def shared_flanks(reads, ref, P):
    """the oracle's insertion pairs (p - 1, p), (p, p + 1) of one read: [(p, first in window, second in window)]"""
    cache, _, _ = O.process_reads(reads, {"R": ref}, ["R"], P, O.make_matrix())
    out = []
    for v in cache.values():
        p = v["variant_R"]
        flat, win = p["all_insertion_positions"], set(map(tuple, p["insertion_coordinates"]))
        pairs = [(flat[k], flat[k + 1]) for k in range(0, len(flat), 2)]
        out += [(a[1], a in win, b in win) for a, b in zip(pairs, pairs[1:]) if a[1] == b[0]]
    return out


@pytest.mark.parametrize("legacy", [False, True])
def test_insertions_sharing_a_flank(eng, legacy):
    """Two insertions around one reference base share that base as a flank; the INS vector counts the shared flank once
    (flank_win in CLASSIFY, win_r / win_l in the general kernel).  Gap open -1 against extend -5 makes the aligner keep
    single-base insertions apart, so reads with bases inserted on both sides of a window edge give pairs with one side in the
    window and the other out, and both in."""
    engine, gpu = eng
    rng = np.random.default_rng(17)
    I = 120
    amp = amplicon(rng, I)
    runs = [(30, 45), (47, 47), (60, 90)]
    ref = window_ref(amp, runs)
    P = O.Params(needleman_wunsch_gap_open=-1, needleman_wunsch_gap_extend=-5, use_legacy_insertion_quantification=legacy)
    reads = []
    for b in boundaries(runs, I):
        for q in (b - 1, b, b + 1):
            if 1 <= q and q + 1 <= I - 1:
                reads.append(amp[:q] + other(rng, amp[q - 1], amp[q]) + amp[q] + other(rng, amp[q], amp[q + 1]) + amp[q + 1:])
                reads.append(amp[:q] + "".join(other(rng, amp[q - 1], amp[q]) for _ in range(3)) + amp[q]
                             + "".join(other(rng, amp[q], amp[q + 1]) for _ in range(2)) + amp[q + 1:])
    sf = shared_flanks(reads, ref, P)
    assert any(x != y for _, x, y in sf) and any(x and y for _, x, y in sf), sf
    reads += [rc(r) for r in reads[::4]]
    SH.run_shape(engine, ref, reads * (4 if gpu else 1), params=P)


@pytest.mark.parametrize("I", [40, 250])
def test_legacy_end_rules_on_window_edges(eng, I):
    """--use_legacy_insertion_quantification reports a deletion starting in alignment column 0 or 1 from reference position 0
    and one reaching the last column up to I - 1: window {0} with a deletion of position 1 is in the window only under
    legacy, as is window {I - 1} with a deletion of the last two positions, and a one-flank insertion on a window edge.
    (The aligner moves a deletion after one leading base to the front, so column 1 is reached through the single-pair
    entry, test_single_pair_entry.)"""
    engine, gpu = eng
    rng = np.random.default_rng(I + 3)
    amp = "ACTG" + SH.rand_seq(rng, I - 8) + "CAGT"                  # no repeat at the ends: the end deletions cannot shift
    reads = [amp[:1] + amp[2:], amp[:1] + amp[3:], amp[1:], amp[2:], amp[:-1], amp[:-2], amp[:-3] + amp[-1:],
             insert_at(rng, amp, 1, 2), insert_at(rng, amp, I - 1, 1), insert_at(rng, amp, I // 2, 3)]
    reads += [rc(r) for r in reads]
    m = O.make_matrix()
    differ = 0
    for runs in ([(0, 0)], [(1, 1)], [(I - 1, I - 1)], [(I - 2, I - 2)], [(0, 0), (I - 1, I - 1)], [(I // 2, I // 2)]):
        ref = window_ref(amp, runs, min_aln_score=40 if I < 64 else 60)
        n_new = O.process_reads(reads, {"R": ref}, ["R"], O.Params(), m)[0]
        n_leg = O.process_reads(reads, {"R": ref}, ["R"], O.Params(use_legacy_insertion_quantification=True), m)[0]
        mods = lambda v: (v["variant_R"]["deletion_n"] > 0, v["variant_R"]["insertion_n"] > 0)
        differ += sum(mods(n_leg[s]) != mods(n_new[s]) for s in n_new)
        for legacy in (False, True):
            P = O.Params(use_legacy_insertion_quantification=legacy)
            PU.check_against_oracle(engine, {"Reference": ref}, ["Reference"], P, reads * (8 if gpu else 1), m)
    assert differ >= 4, differ                                      # the two rules disagree on these windows


# ------------------------------------------------------------------------------------------------ (2) several amplicons
def _block(engine, refs, names, P, reads):
    """process_fastq + quantify -> the count block"""
    import tempfile
    d = tempfile.mkdtemp()
    fq = os.path.join(d, "r.fastq")
    with open(fq, "w") as fh:
        for k, s in enumerate(reads):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))
    cache = {}
    core.process_fastq(fq, cache, names, refs, PU.args_from({k: getattr(P, k) for k in vars(P)}), [], d, engine=engine,
                       aln_matrix=O.make_matrix())
    return core.quantify(cache)


def allele_set(rng, I=200, n=3):
    """WT, an HDR-like allele with a 2-bp insertion inside one of WT's window runs, a SNP allele, and for n = 5 two more SNP
    alleles; each with its own window (four runs; both ends; empty; whole; single positions) -> (refs, names, seqs)"""
    amp = amplicon(rng, I)
    hdr = amp[:100] + "GA" + amp[100:]
    seqs = [amp, hdr, amp[:60] + other(rng, amp[60]) + amp[61:]]
    seqs += [amp[:140] + other(rng, amp[140]) + amp[141:], amp[:30] + other(rng, amp[30]) + amp[31:]][:n - 3]
    windows = [[(40, 50), (52, 60), (63, 70), (90, 110)], [(0, 6), (95, 112), (I - 5, I + 1)], [], [(0, I - 1)],
               [(29, 29), (31, 31), (99, 99), (101, 101)]]
    names = ["WT", "HDR", "SNP", "SNP140", "SNP30"][:n]
    refs = {nm: window_ref(s, w, cut=99) for nm, s, w in zip(names, seqs, windows)}
    return refs, names, seqs


def allele_reads(rng, refs, names, seqs, n_synth):
    reads = []
    for nm, s in zip(names, seqs):
        runs = runs_of(sorted(int(v) for v in refs[nm]["include_idxs"] if 0 <= v < len(s)))
        reads += edge_reads(rng, s, runs)[::2]
        reads += [r.tobytes().decode() for r in synth.synth_reads(rng, s, n_synth, len(s), sub_rate=0.01, rc_frac=0.2,
                                                                   del_frac=0.3, ins_frac=0.2, n_rate=0.002, cut=99)]
    return reads


@pytest.mark.parametrize("n", [3, 5])
def test_amplicons_with_their_own_windows(eng, n):
    """Three amplicons (ALIGN -> CLASSIFY -> general kernel) and five (the general kernel alone), each with its own window
    shape, one of them empty, under expand-ambiguous, assign-first and HDR re-projection, with and without legacy: every
    per-read field, count vector, ref1 vector and histogram against the oracle."""
    engine, gpu = eng
    rng = np.random.default_rng(40 + n)
    refs, names, seqs = allele_set(rng, n=n)
    reads = allele_reads(rng, refs, names, seqs, 64 if gpu else 6)
    m = O.make_matrix()
    sets = [{"expand_ambiguous_alignments": True}, {"assign_ambiguous_alignments_to_first_reference": True},
            {"expected_hdr_amplicon_seq": seqs[1]}, {"expected_hdr_amplicon_seq": seqs[1], "use_legacy_insertion_quantification": True}]
    if not gpu and n > 3:                                  # the emulator's one-kernel form is slow: half the reads, two flag sets
        reads, sets = reads[::2], sets[::3]
    for kw in sets:
        P = O.Params(**kw)
        RS.check_plan(engine, refs, names, reads, m, flags=RS.flags_of(P))
        PU.check_against_oracle(engine, refs, names, P, reads, m)


@pytest.mark.parametrize("legacy", [False, True])
def test_ref1_block_ignores_windows(eng, legacy):
    """The HDR re-projection classifies a read's alignment to reference 0 against reference 0's window but keeps only the
    all_* vectors (CRISPRessoCORE.py:4245-4272), so the ref1 block must not move when only reference 0's window changes."""
    engine, gpu = eng
    rng = np.random.default_rng(7 + legacy)
    refs, names, seqs = allele_set(rng)
    reads = allele_reads(rng, refs, names, seqs, 64 if gpu else 8)
    P = O.Params(expected_hdr_amplicon_seq=seqs[1], use_legacy_insertion_quantification=legacy)
    blocks = []
    for w in ([(40, 50), (52, 60), (63, 70), (90, 110)], [], [(0, 199)], [(0, 0), (199, 199)]):
        refs["WT"] = window_ref(seqs[0], w, cut=99)
        B = _block(engine, refs, names, P, reads)
        blocks.append({r: B.vectors_ref1(r) for r in names[1:]})
    assert any(v.any() for v in blocks[0]["HDR"].values())
    for b in blocks[1:]:
        for r in names[1:]:
            for k, v in b[r].items():
                assert (v == blocks[0][r][k]).all(), (r, k)
    PU.check_against_oracle(engine, refs, names, P, reads, O.make_matrix())


# ------------------------------------------------------------------------------------------------ (3) coding sequence
def coding_masks(I, runs):
    """exon / splicing masks whose boundaries lie on the window's run boundaries, one inside, one outside, and at 0 / I - 1"""
    (a0, a1), (b0, b1) = runs[0], runs[-1]
    def m(ex):
        exon = sorted({p for lo, hi in ex for p in range(lo, hi + 1)})
        splice = sorted({q for lo, hi in ex for q in (lo - 2, lo - 1, hi + 1, hi + 2) if 0 <= q < I})
        return exon, splice
    return {"on": m([(a0, a1), (b0, b1)]), "inside": m([(a0 + 1, a1 - 1), (b0 + 1, b1 - 1)]),
            "outside": m([(a0 - 1, a1 + 1), (b0 - 1, b1 + 1)]), "ends": m([(0, a1), (b0, I - 1)])}


@pytest.mark.parametrize("mask", ["on", "inside", "outside", "ends"])
def test_coding_sequence_on_window_edges(eng, mask):
    """--coding_seq with exon and splicing masks on, one inside and one outside the window's run boundaries and reaching 0 and
    I - 1, exon_len_mods summing to 0, +2 and -3: window deletions that partly overlap an exon or cover only splicing sites,
    insertions whose one exon flank is the in-window one, substitutions on the edges."""
    engine, gpu = eng
    rng = np.random.default_rng(sorted(coding_masks(160, [(30, 50), (100, 120)])).index(mask))
    I = 160
    amp = amplicon(rng, I)
    runs = [(30, 50), (53, 80), (100, 120)]
    exon, splice = coding_masks(I, [runs[0], runs[-1]])[mask]
    reads = edge_reads(rng, amp, runs)
    for a, b in ((45, 56), (25, 35), (115, 125), (51, 54), (98, 101), (120, 123)):     # across exon ends, onto splicing sites
        r = delete(amp, a, b)
        if r:
            reads.append(r)
    for q in (31, 32, 49, 50, 101, 119, 120):
        reads.append(insert_at(rng, amp, q, 2))
    reads += [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 64 if gpu else 8, I, sub_rate=0.01, del_frac=0.4,
                                                               ins_frac=0.3, cut=80)]
    m = O.make_matrix()
    for tem in ([0], [2, 0], [-3]):
        ref = window_ref(amp, runs, cut=80)
        ref.update(contains_coding_seq=True, exon_positions=exon, splicing_positions=splice, exon_len_mods=tem)
        for kw in ({}, {"discard_indel_reads": True}):
            PU.check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(**kw), reads, m)


def test_frame_histogram_extremes(eng):
    """A whole-amplicon window with one exon over the whole amplicon: a near-total deletion gives the most negative frame key,
    a long insertion the largest, around hist_zero with tot_exon_len_mod 0, +2 and -3 (c2b_configure's layout reaches
    hist_zero - I - |tem| .. hist_zero + J + |tem|)."""
    engine, gpu = eng
    rng = np.random.default_rng(5)
    I = 40
    amp = amplicon(rng, I)
    long_ins = amp[:20] + "".join(other(rng, amp[19], amp[20]) for _ in range(400)) + amp[20:]
    reads = [amp[:3] + amp[-3:], amp[:4] + amp[-3:], long_ins, amp[:20] + long_ins[20:300] + amp[20:], amp]
    m = O.make_matrix()
    for tem in (0, 2, -3):
        ref = window_ref(amp, [(0, I - 1)], min_aln_score=1)
        ref.update(contains_coding_seq=True, exon_positions=list(range(I)), splicing_positions=[], exon_len_mods=[tem])
        extras = {}
        cache = O.process_reads(reads, {"R": ref}, ["R"], O.Params(), m)[0]
        O.count_vectors(cache, {"R": ref}, ["R"], O.Params(), extras)
        keys = set(extras["R"]["hists_inframe"]) | set(extras["R"]["hists_frameshift"])
        assert min(keys) <= -(I - 6) + tem and max(keys) >= 400 + tem, keys
        PU.check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(), reads, m)


# ------------------------------------------------------------------------------------------------ (4) single-pair entry
@pytest.mark.parametrize("I", [40, 250])
def test_single_pair_entry(eng, I, monkeypatch):
    """resources.find_indels_substitutions / find_indels_substitutions_legacy (c2b_classify_aligned: the general kernel's row
    space on one aligned pair) against the oracle, on the alignments of the edge batches under every window shape, and with
    values outside [0, I) added (-5, -1, I, I + 1, 4 I), which the reference never looks up and the engine must ignore."""
    engine, gpu = eng
    monkeypatch.setattr(resources, "_pair_engine", engine)
    rng = np.random.default_rng(90 + I)
    amp = amplicon(rng, I)
    shapes = window_shapes(I)
    reads = edge_reads(rng, amp, shapes["four_runs"])
    cache = O.process_reads(reads, {"R": window_ref(amp, [])}, ["R"], O.Params(), O.make_matrix())[0]
    pairs = sorted({(v["variant_R"]["aln_seq"], v["variant_R"]["aln_ref"]) for v in cache.values()})
    q = I // 2                                                      # hand-built: two insertions sharing flank q, runs at the ends
    pairs += [(amp[:q] + "A" + amp[q] + "C" + amp[q + 1:], amp[:q] + "-" + amp[q] + "-" + amp[q + 1:]),
              ("-" + amp[1:-1] + "-", amp), ("--" + amp[2:], amp), (amp[0] + "-" + amp[2:], amp),
              (amp[0] + "--" + amp[3:], amp), (amp[:-2] + "--", amp), ("G" + amp + "T", "-" + amp + "-")]
    if not gpu:
        pairs = pairs[::3] + pairs[-5:]
    n = 0
    for name, runs in shapes.items():
        idx = sorted({p for lo, hi in runs for p in range(lo, hi + 1)})
        for inc in (idx, idx + [-5, -1, I, I + 1, 4 * I]):
            for s1, s2 in pairs:
                for fn, want in ((resources.find_indels_substitutions, O.find_indels_substitutions),
                                 (resources.find_indels_substitutions_legacy, O.find_indels_substitutions_legacy)):
                    w = want(s1, s2, [v for v in inc if 0 <= v < I])
                    assert not G.payload_equal(w, fn(s1, s2, inc)), (name, inc[:8], s1, s2)
                    n += 1
    assert n > 200


# ------------------------------------------------------------------------------------------------ (5) annotations
@pytest.mark.parametrize("legacy", [False, True])
def test_annotation_pass_on_window_edges(eng, tmp_path, legacy):
    """--fastq_output / --bam_output annotations (DEL= / INS= / SUB= filter the edit list by in_window; legacy rebuilds deletion
    sizes) against the reference's own process_fastq_write_out / process_single_fastq_write_bam_out, for a window of four
    runs and one touching both ends."""
    engine, gpu = eng
    import annotate_util as AU
    if not AU.have_reference():
        pytest.skip("needs oracle/_ref/install (built by __graft_entry__.build())")
    sys.path.insert(0, os.path.dirname(HERE))
    from baseline import ref_shim
    old_path = os.environ["PATH"]
    os.environ["PATH"] = AU.fake_samtools(str(tmp_path / "bin"))
    try:
        rng = np.random.default_rng(60 + legacy)
        core_mod = ref_shim.load_core()
        I = 250
        amp = amplicon(rng, I)
        fq = AU.write_fastq(str(tmp_path / "w.fastq"), edge_reads(rng, amp, window_shapes(I)["four_runs"]))
        argv = ["-r1", fq, "-a", amp, "-g", amp[110:130]] + (["--use_legacy_insertion_quantification"] if legacy else [])
        ref_names, refs, args = AU.capture(tmp_path, argv)
        for k, runs in enumerate((window_shapes(I)["four_runs"], window_shapes(I)["both_ends"])):
            for r in refs.values():
                r["include_idxs"] = np.array(sorted({p for lo, hi in runs for p in range(lo, hi + 1)}), dtype=np.int64)
            fq2 = AU.write_fastq(str(tmp_path / ("e%d.fastq" % k)), edge_reads(rng, amp, runs))
            d = tmp_path / ("p%d" % k)
            d.mkdir()
            P = AU.Pair(core_mod, engine, d, ref_names, refs, args)
            res_r, res_b, cache_r, cache_b, text_r, text_b, untouched = P.fastq(fq2, "f")
            assert untouched and text_r == text_b and b" DEL=" in text_r
            AU.check_results(res_r, res_b, cache_r, cache_b)
            res_r, res_b, cache_r, cache_b, sam_r, sam_b = P.sam(fq2, "s")
            assert sam_r == sam_b
            AU.check_results(res_r, res_b, cache_r, cache_b)
    finally:
        os.environ["PATH"] = old_path


# ------------------------------------------------------------------------------------------------ (6) large batches, GPU
@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(window_shapes(250)))
def test_large_batch_per_shape(eng, shape):
    """16 Ki reads of a 250-bp amplicon per window shape through the full tier sequence: the one-length part and the whole
    batch each run with every shortcut on, with C2B_NO_DIAG + C2B_NO_NARROW, with C2B_NO_SPLIT and with every shortcut off,
    and must compute the same (SH.run_shape); 3 Ki of them against the oracle."""
    engine, gpu = eng
    if not gpu:
        pytest.skip("GPU-sized batch")
    rng = np.random.default_rng(7000 + sorted(window_shapes(250)).index(shape))
    I = 250
    amp = amplicon(rng, I)
    runs = window_shapes(I)[shape]
    ref = window_ref(amp, runs)
    edge = edge_reads(rng, amp, runs)
    synth_reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 16384 - 4 * len(edge), I, sub_rate=0.01,
                                                                    rc_frac=0.2, del_frac=0.3, ins_frac=0.2, n_rate=0.002,
                                                                    cut=int(rng.integers(20, I - 20)))]
    reads = edge * 4 + synth_reads
    reads = [reads[i] for i in rng.permutation(len(reads))]
    assert len(reads) == 16384
    adm, cnt = SH.run_shape(engine, ref, [r for r in reads if len(r) == I], oracle=False)
    assert cnt["diag"][0] > 0, cnt
    SH.run_shape(engine, ref, reads, oracle=False)
    PU.check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(), edge + reads[:3072 - len(edge)],
                            O.make_matrix())
