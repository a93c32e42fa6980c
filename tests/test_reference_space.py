"""The engine against the oracle over the reference space: the set of amplicons every read is tried against.

The amplicon count decides which device code runs (DESIGN.md section 3): up to RG_MAX_REFS = 4 amplicons that all admit the
packed DP take the two-kernel form (ALIGN -> CLASSIFY, then the general kernel over the left-overs); 5 to C2B_MAX_REFS = 32
amplicons, or 2-4 where one carries a coding sequence, run the general kernel alone, whose phase sets move in step on named
barriers (3 + 4 * (3 + 2 * n_refs) per work group) and keep one op stream per reference in `opsbuf`.  Each reference also
has its own admission: the ring needs the read within RG_MAXD = 8 bases of that amplicon and the amplicon inside one 256-row
block, the packed DP needs the read within that amplicon's pk_maxJ, and the string width W comes from the longest amplicon.

`allele_panel()` builds n variants of one amplicon (SNPs, small indels, long exact shared stretches) so that reads tie
across chosen subsets of the panel.  Every batch goes through the oracle (PU.check_against_oracle: per-read fields,
aln_stats, every count vector, scalar and histogram, ref1 vectors under HDR), and the launch sequence that plan_batch
predicts is checked with launch_count() / path_counts() / ring_counts(), so a test fails when it ran another path than the
one it names.  Slot independence (CRISPRessoCORE.py:656-707 aligns each reference on its own): slot r of an n-amplicon batch
must equal a one-amplicon batch against amplicon r, which needs no oracle and so runs at 16 Ki reads on the GPU.

Runs on the CPU warp emulator with small batches; with -m gpu the same checks run through the sm_90a library, larger."""
import os
import sys

import numpy as np
import pytest

import parity_util as PU
import test_shape_space as SH
from crispresso2_b200 import _lib, core, synth
from crispresso2_b200.engine import Engine, EngineError, pack_reads
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ACGT = list("ACGT")
MAX_REFS, MAX_POOLED, RG_MAX_REFS = 32, 1024, 4          # C2B_MAX_REFS, C2B_MAX_POOLED_REFS (include/c2b200.h), c2b_core.cuh
COUNTS = [2, 4, 5, 6, 8, 16, 31, 32]
FLAG_SETS = [("plain", {}), ("expand", {"expand_ambiguous_alignments": True}),
             ("assign_first", {"assign_ambiguous_alignments_to_first_reference": True}), ("hdr", None),
             ("discard_indel", {"discard_indel_reads": True}),
             ("ignore", {"ignore_substitutions": True, "ignore_insertions": True, "ignore_deletions": True})]


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def eng(request):
    """(engine, on_gpu): the warp-emulator build with small batches; with -m gpu the sm_90a library on cuda:0"""
    if request.param == "gpu":
        return Engine(0), True
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import build_emu
    return Engine(lib_path=build_emu.build()), False


def new_engine(engine):
    """a fresh engine on the same build"""
    return Engine(0) if engine.lib_path is None else Engine(lib_path=engine.lib_path)


rc = SH.rc


def rand_seq(rng, n):
    return "".join(rng.choice(ACGT, n))


# ------------------------------------------------------------------------------------------------ the panel
def allele_panel(rng, n, L=200, guide=(85, 115)):
    """n allele variants of one random L-bp amplicon.  Allele k carries one edit at its own site, outside the guide window
    `guide` and 8 bp from either end; everything else is shared exactly.  Edits: a SNP, except a 1-bp deletion for k % 4 == 3
    and a 3-bp insertion for k % 8 == 6 (so the last allele of 4, 8, 16 or 32 is a deletion and ties).  So the amplicon itself scores (L - 1) / L against every SNP and 1-bp-deletion
    allele (a tie across all of them), and a read carrying the edits of SNP alleles S ties across exactly S.
    -> (base amplicon, [allele sequences], [(site, kind)])"""
    base = rand_seq(rng, L)
    free = [p for p in range(8, L - 8) if not guide[0] - 2 <= p < guide[1] + 2]
    sites = [free[int(round(x))] for x in np.linspace(0, len(free) - 1, n)]
    seqs, edits = [], []
    for k, p in enumerate(sites):
        kind = "ins" if k % 8 == 6 else ("del" if k % 4 == 3 else "snp")
        if kind == "snp":
            s = base[:p] + rng.choice([c for c in ACGT if c != base[p]]) + base[p + 1:]
        elif kind == "del":
            s = base[:p] + base[p + 1:]
        else:
            s = base[:p] + rand_seq(rng, 3) + base[p:]
        seqs.append(s)
        edits.append((p, kind))
    return base, seqs, edits


def with_edits(base, seqs, edits, ks):
    """the base amplicon with the edits of alleles ks applied (right to left, so that sites stay put)"""
    s = base
    for k in sorted(ks, key=lambda k: -edits[k][0]):
        p, kind = edits[k]
        a = seqs[k]
        s = s[:p] + a[p:p + (1 if kind == "snp" else 3 if kind == "ins" else 0)] + s[p + 1 if kind != "ins" else p:]
    return s


def panel_refs(seqs, names=None, cut=99, min_scores=None, seed_len=10):
    names = names or ["A%02d" % k for k in range(len(seqs))]
    refs = {}
    for k, (nm, s) in enumerate(zip(names, seqs)):
        refs[nm] = SH.shape_ref(s, seed_len=seed_len, cut=min(cut, len(s) - 2), window=3,
                                min_aln_score=60 if min_scores is None else min_scores[k])
    return refs, names


def thresholds(base, seqs, edits, rng, m):
    """per-amplicon min_aln_score (the CLI's -amas), and the reads that sit on them: for amplicon k a read that is allele k
    with a few substitutions and a threshold just below (k % 3 == 0), exactly at (1: the strict test fails) or just above (2)
    its score; amplicon 1's threshold is the score of the read that ties amplicons 0 and 1, so amplicon 1 joins the winners
    only through the equality branch of CRISPRessoCORE.py:697-707 -> (min scores, threshold reads)"""
    mins, reads = [], []
    for k, s in enumerate(seqs):
        t = list(s)
        for p in rng.choice(len(s), 6, replace=False):
            t[p] = rng.choice([c for c in ACGT if c != t[p]])
        t = "".join(t)
        sc = O.global_align(t, s, m, SH.shape_ref(s)["gap_incentive"], -20, -2)[2]
        mins.append(round(sc + (-0.001, 0.0, 0.001)[k % 3], 3))
        reads.append(t)
    snps = [k for k, e in enumerate(edits) if e[1] == "snp"]
    if len(snps) >= 2 and snps[:2] == [0, 1]:
        tie = with_edits(base, seqs, edits, [0, 1])
        mins[1] = O.global_align(tie, seqs[1], m, SH.shape_ref(seqs[1])["gap_incentive"], -20, -2)[2]
        reads += [tie, tie]
    return mins, reads


def panel_reads(rng, base, seqs, edits, budget):
    """copies of every allele; the base amplicon (ties every SNP / deletion allele); reads that tie 2 and 3 SNP alleles;
    reverse complements, N bases, substitutions, reads that match no amplicon -- at most `budget` reads"""
    snps = [k for k, e in enumerate(edits) if e[1] == "snp"]
    two = [with_edits(base, seqs, edits, snps[j:j + 2]) for j in range(0, len(snps) - 1, 2)]
    three = [with_edits(base, seqs, edits, snps[j:j + 3]) for j in range(0, len(snps) - 2, 3)]
    out = [base, rc(base)] + two[:1] + three[:1] + list(seqs[:2]) + two[1:] + three[1:]
    out += list(seqs[2:]) + [rc(s) for s in seqs[::3]]
    for s in seqs[1::4]:
        p = int(rng.integers(0, len(s)))
        out.append(s[:p] + "N" + s[p + 1:])
    out += [rand_seq(rng, len(base)), rand_seq(rng, len(base) - 17)]
    out += [s[:60] + rand_seq(rng, 20) + s[80:] for s in seqs[2::5]]
    head = out[:6]
    rest = out[6:]
    while len(head) + len(rest) < budget:                  # alleles with a few substitutions
        t = list(seqs[int(rng.integers(0, len(seqs)))])
        for p in rng.choice(len(t), int(rng.integers(1, 4)), replace=False):
            t[p] = rng.choice(ACGT)
        rest.append("".join(t))
    order = rng.permutation(len(rest))
    return (head + [rest[i] for i in order])[:budget]


def flags_of(params):
    return core._flags(PU.args_from({k: getattr(params, k) for k in vars(params)}))


# ------------------------------------------------------------------------------------------------ the launch sequence
def launches_of(engine, refs, names, reads, m, flags=0):
    """one engine-level batch -> (kernel launches, path_counts, ring_counts, result)"""
    engine.configure(refs, names, m, -20, -2, 5, 2, flags, "ACGTN", 48)
    engine.counts_reset()
    before = engine.launch_count()
    res = engine.align(reads)
    n = engine.launch_count() - before
    return n, engine.path_counts(), engine.ring_counts(), res


def check_plan(engine, refs, names, reads, m, flags=0, one_kernel=None):
    """plan_batch's choice for every read tried against every amplicon: ALIGN, CLASSIFY and the general kernel up to
    RG_MAX_REFS amplicons that all admit the packed DP, else the general kernel alone over every pair of reads"""
    n_refs = len(names)
    if one_kernel is None:
        one_kernel = n_refs > RG_MAX_REFS
    launches, (pairs, singles), ring, res = launches_of(engine, refs, names, reads, m, flags)
    if one_kernel:                                     # its groups try the ring only up to RG_MAX_REFS amplicons
        assert launches == 1 and pairs + singles == (len(reads) + 1) // 2, (n_refs, launches, pairs, singles)
        assert ring == (0, 0) or n_refs <= RG_MAX_REFS, (n_refs, ring)
    else:
        assert launches == 3, (n_refs, launches)
        if len(reads) >= 16:                              # ALIGN's groups of eight took some pairs
            assert sum(ring) > 0, ring
    return res


# ------------------------------------------------------------------------------------------------ (1) count sweep
@pytest.mark.parametrize("n", COUNTS)
def test_count_sweep(eng, n):
    """n allele amplicons under no flag, expand-ambiguous, assign-first, HDR re-projection of every other amplicon onto
    amplicon 0, discard-indel and the three ignore flags; per-amplicon thresholds with reads on them.  The emulator runs
    every flag set up to 5 amplicons, three at 6 and 8 and one above, rotating with n; the GPU runs all of them with more
    reads."""
    engine, gpu = eng
    rng = np.random.default_rng(500 + n)
    m = O.make_matrix()
    base, seqs, edits = allele_panel(rng, n)
    mins, treads = thresholds(base, seqs, edits, rng, m)
    refs, names = panel_refs(seqs, min_scores=mins)
    budget = (3 * n + 40) if gpu else max(16, min(3 * n + 8, 640 // n))
    reads = panel_reads(rng, base, seqs, edits, budget) + treads[:budget // 3]
    if gpu:
        reads += [r.tobytes().decode() for s in seqs[:4] for r in synth.synth_reads(rng, s, 64, len(s), sub_rate=0.01, rc_frac=0.2,
                                                                                    del_frac=0.2, ins_frac=0.1, n_rate=0.002, cut=99)]
    # the oracle sees the tie structure the panel promises
    cache_o = O.process_reads(reads, refs, names, O.Params(), m)[0]
    ties = {len(v["aln_ref_names"]) for v in cache_o.values()}
    assert {2, 3} <= ties or n == 2 and 2 in ties, ties
    assert any(len(v["aln_ref_names"]) == sum(1 for e in edits if e[1] != "ins") for v in cache_o.values())
    assert any(mins[1] == v["aln_scores"][1] and names[1] in v["aln_ref_names"] for v in cache_o.values())
    sets = FLAG_SETS if gpu or n <= 5 else [FLAG_SETS[(n + k) % 6] for k in ((0, 2, 4) if n <= 8 else (0,))]
    for name, kw in sets:
        P = O.Params(expected_hdr_amplicon_seq=seqs[1]) if kw is None else O.Params(**kw)
        check_plan(engine, refs, names, reads, m, flags_of(P))
        PU.check_against_oracle(engine, refs, names, P, reads, m)


# ------------------------------------------------------------------------------------------------ (2) slot independence
def compact_run(engine, refs, names, reads, m):
    engine.configure(refs, names, m, -20, -2, 5, 2, 0, "ACGTN", 48)
    engine.counts_reset()
    buf, off = pack_reads(reads)
    n = len(reads)
    return engine.align_packed(buf, off, compact=True, count=np.ones(n, dtype=np.int32), qweight=np.ones(n, dtype=np.int32))


CLASS_FIELDS = ("n_edits", "insertion_n", "deletion_n", "substitution_n", "n_ins_all", "n_ins_win", "n_del_all", "n_del_win",
                "n_del_pos_all", "n_sub_all", "irregular_ends", "modified")


def check_slots(engine, refs, names, reads, m, strings_for=64):
    """slot r of the n-amplicon batch == the one-amplicon batch against amplicon r: score, strand, columns, op stream and the
    aligned strings of every read; classification fields and edit lists where amplicon r wins in both"""
    ns = min(strings_for, len(reads))
    multi = compact_run(engine, refs, names, reads, m)
    assert int(multi.alns.shape[1]) == len(names)
    ms = multi.strings_block(0, ns)                       # rebuilt against the configuration that aligned them
    winners = 0
    for r, nm in enumerate(names):
        one = compact_run(engine, {nm: refs[nm]}, [nm], reads, m)
        os1 = one.strings_block(0, ns)
        a, b = multi.alns[:, r], one.alns[:, 0]
        for f in ("score_milli", "strand", "aln_len", "n_match", "status"):
            assert (a[f] == b[f]).all(), (nm, f, np.nonzero(a[f] != b[f])[0][:8])
        assert ((multi.meta[:, r] & 0xffffff) == (one.meta[:, 0] & 0xffffff)).all(), nm
        cols = (one.meta[:, 0] & 0xffff).astype(np.int64)
        for k in range(len(reads)):
            used = (int(cols[k]) + 31) // 32
            assert (multi.ops[k, r, :used] == one.ops[k, 0, :used]).all(), (nm, k)
        for k in range(ns):
            w = int(b["aln_len"][k])
            assert (ms[k, r, :, multi.W - w:] == os1[k, 0, :, one.W - w:]).all(), (nm, k)
        win = (((multi.recs["winner_mask"].astype(np.int64) >> (r & 31)) & 1) != 0) & (multi.recs["best_score_milli"] > 0) \
            & (one.recs["best_score_milli"] > 0)
        winners += int(win.sum())
        for f in CLASS_FIELDS:
            assert (a[f][win] == b[f][win]).all(), (nm, f)
        ea, fa = PU.edits_canonical(multi, r)
        eb, fb = PU.edits_canonical(one, 0)
        assert (fa[win] == fb[win]).all() and (ea[win & fa] == eb[win & fb]).all(), nm
    assert winners > 0
    return multi


@pytest.mark.parametrize("n", [5, 8, 32])
def test_slot_independence(eng, n):
    """Each amplicon's alignment does not depend on the others: a warp of a phase set that read another warp's opsbuf slice,
    or a reference loop cut short, changes some slot.  GPU: 16 Ki reads x 8 amplicons and 4 Ki reads x 32 amplicons, with
    an oracle subset of a few hundred reads; the emulator runs a small batch."""
    engine, gpu = eng
    rng = np.random.default_rng(900 + n)
    m = O.make_matrix()
    base, seqs, edits = allele_panel(rng, n)
    refs, names = panel_refs(seqs)
    pool = panel_reads(rng, base, seqs, edits, 4 * n + 16 if gpu else {5: 24, 8: 20, 32: 12}[n])
    if gpu:
        total = {5: 4096, 8: 16384, 32: 4096}[n]
        extra = [r.tobytes().decode() for r in synth.synth_reads(rng, base, total - len(pool), len(base), sub_rate=0.01, rc_frac=0.2,
                                                                 del_frac=0.2, ins_frac=0.1, n_rate=0.002, cut=99)]
        reads = pool + extra
    else:
        reads = pool
    check_slots(engine, refs, names, reads, m, strings_for=256 if gpu else 64)
    PU.check_against_oracle(engine, refs, names, O.Params(expand_ambiguous_alignments=True), reads[:(300 if gpu else 12)], m)


# ------------------------------------------------------------------------------------------------ (3) mixed lengths
def mixed_sets(rng):
    """(label, amplicon sequences, read lengths, whether every amplicon admits the ring-banded two-kernel form)"""
    a = rand_seq(rng, 200)
    b256 = rand_seq(rng, 256)
    long = rand_seq(rng, 700)
    return [
        # a read of 200 is 0 / 8 / 9 away from these amplicons; reads of 191 / 192 / 208 / 209 straddle the other edges
        ("rg_maxd", [a, a[:100] + rand_seq(rng, 8) + a[100:], a[:100] + rand_seq(rng, 9) + a[100:], a[:95] + a[104:]],
         [200, 191, 192, 208, 209]),
        # one row block and two
        ("row_blocks", [b256, b256[:128] + "G" + b256[128:], b256[:200]], [256, 257, 250, 248]),
        # W from the 700-bp amplicon; I + J against it reaches C2B_MAX_ALN_LEN = 1024 columns at J = 324
        ("short_long", [a[:60], long, a[:60] + "T" + a[60:120]], [60, 61, 120, 323, 324]),
    ]


@pytest.mark.parametrize("label", ["rg_maxd", "row_blocks", "short_long", "pk_maxj", "rg_maxd_5"])
def test_mixed_amplicon_lengths(eng, label):
    """Amplicon sets whose per-reference admission differs for one read: the ring's RG_MAXD, one and two 256-row blocks, a
    60-bp amplicon beside a 700-bp one, amplicons with different pk_maxJ (a large gap incentive at one amplicon's cut), and
    the RG_MAXD set with five amplicons (one-kernel form).  On the RG_MAXD set the ring runs, and both ring results and
    full-matrix fallbacks must occur."""
    engine, gpu = eng
    rng = np.random.default_rng(sum(map(ord, label)))
    m = O.make_matrix()
    per = 8 if gpu else 2
    if label == "pk_maxj":
        import test_scoring_space as SS
        a = rand_seq(rng, 200)
        seqs = [a, a[:120] + "C" + a[121:]]
        refs, names = panel_refs(seqs)
        gi = np.zeros(201, dtype=np.int64)
        gi[100] = 16                                    # pk_maxJ 170 or so (at 40 the packed DP is refused outright)
        refs[names[1]]["gap_incentive"] = gi
        pk = [SS.admission(m, seqs[k], refs[names[k]]["gap_incentive"], -20, -2)["pk_maxJ"] for k in range(2)]
        assert 0 < pk[1] < 200 < pk[0], pk
        lens = [pk[1] - 1, pk[1], pk[1] + 1, 200]
        one_kernel = False
    else:
        sets = {s[0]: s for s in mixed_sets(rng)}
        _, seqs, lens = sets["rg_maxd" if label == "rg_maxd_5" else label]
        if label == "rg_maxd_5":
            seqs = seqs + [seqs[0][:150] + "A" + seqs[0][151:]]
        refs, names = panel_refs(seqs, cut=30 if label == "short_long" else 99)
        one_kernel = len(seqs) > RG_MAX_REFS
    reads = []
    for J in lens:
        for s in seqs:
            reads += SH.shape_reads(rng, s, J, per)
    if label == "pk_maxj":                              # full groups of the amplicon's length, where the ring runs
        reads += SH.shape_reads(rng, seqs[0], 200, 2 * per) + [seqs[0]] * 8
    if label == "short_long":
        assert max(len(r) for r in reads) + max(len(s) for s in seqs) == 1024
    res = check_plan(engine, refs, names, reads, m, one_kernel=one_kernel)
    ring = engine.ring_counts()
    if label == "rg_maxd":
        assert ring[0] > 0 and ring[1] > 0, ring
    assert res.W == ((max(len(s) for s in seqs) + max(len(r) for r in reads) + 31) & ~31)
    PU.check_against_oracle(engine, refs, names, O.Params(expand_ambiguous_alignments=True), reads, m)
    if gpu or label != "short_long":
        check_slots(engine, refs, names, reads[:(len(reads) if gpu else 16)], m)


# ------------------------------------------------------------------------------------------------ (4) coding sequence
@pytest.mark.parametrize("n", [2, 3, 4, 6])
def test_coding_sequence_on_some_amplicons(eng, n):
    """--coding_seq that lies in one amplicon of the set (exon and splicing positions there, none elsewhere): split_all is
    false, so even 2-4 amplicons run the one-kernel form."""
    engine, gpu = eng
    rng = np.random.default_rng(40 + n)
    m = O.make_matrix()
    base, seqs, edits = allele_panel(rng, n)
    refs, names = panel_refs(seqs)
    c = names[n // 2]
    refs[c].update(contains_coding_seq=True, exon_positions=list(range(40, 90)) + list(range(120, 160)), exon_len_mods=[0, 0],
                   splicing_positions=[38, 39, 90, 91, 118, 119, 160, 161])
    reads = panel_reads(rng, base, seqs, edits, 40 if gpu else 14)
    reads += [r.tobytes().decode() for r in synth.synth_reads(rng, seqs[n // 2], 200 if gpu else 10, len(seqs[n // 2]), sub_rate=0.02,
                                                             del_frac=0.35, ins_frac=0.25, rc_frac=0.1, cut=99)]
    check_plan(engine, refs, names, reads, m, one_kernel=True)
    for kw in ({}, {"expand_ambiguous_alignments": True, "expected_hdr_amplicon_seq": seqs[1]}):
        PU.check_against_oracle(engine, refs, names, O.Params(**kw), reads, m)


# ------------------------------------------------------------------------------------------------ (5) seed tests
def test_seed_tests_disagree_across_six_amplicons(eng):
    """Six amplicons whose seed tests disagree for one read: two seeded amplicons and an allele of the first, an amplicon too
    short for any seed, a reverse-complement-symmetric one (every k-mer in its reverse complement: no seed), and a seeded
    amplicon sharing only its ends with the first.  Reads are forward for some amplicons and both-strand for others, and
    the construction of PU.check_seed_disagreement (the front of a forward read joined to the reverse complement of its
    back half) runs over the whole set."""
    engine, gpu = eng
    rng = np.random.default_rng(606)
    m = O.make_matrix()
    a = rand_seq(rng, 160)
    half = rand_seq(rng, 80)
    seqs = {"A": a, "A2": a[:70] + "T" + a[71:], "B": rand_seq(rng, 160), "SHORT": a[50:84], "SYM": half + rc(half),
            "ENDS": a[:20] + rand_seq(rng, 120) + a[140:]}
    names = list(seqs)
    refs = {k: SH.shape_ref(s, exclude=12 if k == "SHORT" else None) for k, s in seqs.items()}
    assert refs["SHORT"]["fw_seeds"] == [] and refs["SYM"]["fw_seeds"] == [] and refs["A"]["fw_seeds"] and refs["B"]["fw_seeds"]
    n = 96 if gpu else 12
    reads = []
    for s in (a, seqs["B"], seqs["ENDS"], seqs["SYM"]):
        reads += [r.tobytes().decode() for r in synth.synth_reads(rng, s, n // 4, len(s), sub_rate=0.01, rc_frac=0.3, cut=80)]
    reads += [r[:80] + rc(r)[:80] for r in reads[0:n // 2:2]]
    reads += [rc(r) for r in reads[1:n // 2:2]]
    P = O.Params()
    modes = [tuple(O._strand_choice(P, s, refs[r]) for r in names) for s in reads]
    assert sum(1 for md in modes if "fw" in md and "both" in md) >= len(reads) // 4
    assert sum(1 for md in modes if "rc" in md and "both" in md) >= 2
    check_plan(engine, refs, names, reads, m)
    for kw in ({}, {"expand_ambiguous_alignments": True}):
        PU.check_against_oracle(engine, refs, names, O.Params(**kw), reads, m)


# ------------------------------------------------------------------------------------------------ (6) re-configuration
def test_reconfigure_one_engine(eng):
    """One engine configured through 32, 2, 17, 5, 4, 1 and 32 amplicons with growing and shrinking read lengths: opsbuf and
    the other scratch buffers are sized from n_refs and the read length, and every step must equal a fresh engine's."""
    engine, gpu = eng
    rng = np.random.default_rng(3217)
    m = O.make_matrix()
    base, seqs, edits = allele_panel(rng, 32, L=180)
    steps = [(32, 150), (2, 260), (17, 120), (5, 300), (4, 180), (1, 240), (32, 100)]
    n = 128 if gpu else 6
    for k, (nr, J) in enumerate(steps):
        sel = [seqs[(3 * k + j) % 32] for j in range(nr)]
        refs, names = panel_refs(sel, names=["R%d_%d" % (k, j) for j in range(nr)])
        pool = panel_reads(rng, base, sel, [edits[(3 * k + j) % 32] for j in range(nr)], n - 1)
        reads = [(s + rand_seq(rng, J))[:J] for s in pool] + [rand_seq(rng, J)]
        got = SH._run(engine, refs, names, reads, O.Params(), m)
        fresh = new_engine(engine)
        want = SH._run(fresh, refs, names, reads, O.Params(), m)
        fresh.close()
        SH.same_results(got[0], got[1], want[0], want[1])
        assert got[2] == want[2], (k, got[2], want[2])


# ------------------------------------------------------------------------------------------------ (7) chunked pipeline
@pytest.mark.parametrize("n", [5, 32])
def test_chunked_pipeline_many_amplicons(eng, monkeypatch, n):
    """c2b_align_batch splits a batch into pipelined chunks (C2B_CHUNK) through pinned bounce buffers (C2B_FORCE_BOUNCE):
    5- and 32-amplicon batches, full and compact outputs, must equal one chunk."""
    engine, gpu = eng
    rng = np.random.default_rng(70 + n)
    m = O.make_matrix()
    base, seqs, edits = allele_panel(rng, n)
    refs, names = panel_refs(seqs)
    reads = panel_reads(rng, base, seqs, edits, 200 if gpu else (23 if n == 5 else 11))
    reads[3] = reads[3][:150]
    out = []
    for chunk, bounce, compact in ((None, "0", False), ("7", "0", False), ("7", "1", False), ("9", "1", True), (None, "1", True)):
        if chunk:
            monkeypatch.setenv("C2B_CHUNK", chunk)
        else:
            monkeypatch.delenv("C2B_CHUNK", raising=False)
        monkeypatch.setenv("C2B_FORCE_BOUNCE", bounce)
        engine.configure(refs, names, m, -20, -2, 5, 2, 0, "ACGTN", 16)
        engine.counts_reset()
        buf, off = pack_reads(reads)
        out.append((engine.align_packed(buf, off, compact=compact), engine.counts_raw()))
    monkeypatch.delenv("C2B_CHUNK", raising=False)
    monkeypatch.delenv("C2B_FORCE_BOUNCE", raising=False)
    a, ca = out[0]
    for b, cb in out[1:]:
        assert (a.recs == b.recs).all() and (a.alns == b.alns).all() and (ca == cb).all()
        for r in range(n):
            (ea, fa), (eb, fb) = PU.edits_canonical(a, r), PU.edits_canonical(b, r)
            assert (fa == fb).all() and (ea[fa] == eb[fb]).all()
        for i in range(len(reads)):
            for r in (0, n // 2, n - 1):
                assert a.pair(i, r) == b.pair(i, r)


# ------------------------------------------------------------------------------------------------ (8) annotations
def _annotation_env():
    import annotate_util as AU
    if not AU.have_reference():
        pytest.skip("needs oracle/_ref/install (built by __graft_entry__.build())")
    return AU


@pytest.mark.parametrize("n", [6, 32])
def test_annotations_many_amplicons(eng, tmp_path, n):
    """--fastq_output / --bam_output annotations and the process_bam "c2:Z:" form against the reference's own wrappers, with
    the (ref_names, refs, args) its main() builds for `-a` with n allele amplicons; ALN_DETAILS lists every amplicon.  The
    annotation pass is also run in chunks of 5 reads, which must give the same bytes."""
    engine, gpu = eng
    AU = _annotation_env()
    import bam_util as BU
    import test_bam_input as TB
    from crispresso2_b200 import annotate
    from baseline import ref_shim
    rng = np.random.default_rng(60 + n)
    base, seqs, edits = allele_panel(rng, n)
    reads = panel_reads(rng, base, seqs, edits, (3 * n + 20) if gpu else (16 if n == 6 else 10))
    fq = AU.write_fastq(str(tmp_path / "panel.fastq"), reads)
    old_path = os.environ["PATH"]
    os.environ["PATH"] = BU.fake_samtools(str(tmp_path / "bin"))
    try:
        ref_names, refs, args = AU.capture(tmp_path, ["-r1", fq, "-a", ",".join(seqs), "-g", base[90:110],
                                                      "--expand_ambiguous_alignments"])
        assert len(ref_names) == n
        core_mod = ref_shim.load_core()
        d = tmp_path / "p"
        d.mkdir()
        P = AU.Pair(core_mod, engine, d, ref_names, refs, args)
        res_r, res_b, cache_r, cache_b, text_r, text_b, untouched = P.fastq(fq, "f")
        assert untouched and text_r == text_b and text_r.count(b"\n") >= 4
        AU.check_results(res_r, res_b, cache_r, cache_b)
        assert any(len(v["aln_ref_names"]) > 2 for v in cache_r.values())
        whole = annotate.Annotation(cache_b, refs)
        parts = annotate.Annotation(cache_b, refs, chunk=5)
        assert (whole.ann_off == parts.ann_off).all() and bytes(whole.arena) == bytes(parts.arena)
        res_r, res_b, cache_r, cache_b, sam_r, sam_b = P.sam(fq, "s")
        assert sam_r == sam_b
        AU.check_results(res_r, res_b, cache_r, cache_b)
        bam_path = TB.write_synthetic(str(tmp_path / "panel.bam"), reads)
        env = {"CORE": core_mod, "engine": engine, "tmp": tmp_path, "caps": {"panel": (ref_names, refs, args)}}
        _, _, _, sam = TB.check_both(env, "panel", bam_path, "", "bam", samtools_exclude_flags="4")
        assert sam.count(b"\tc2:Z:") >= 4
    finally:
        os.environ["PATH"] = old_path


# ------------------------------------------------------------------------------------------------ (9) limits
def _fastq(tmp_path, reads):
    fq = tmp_path / "r.fastq"
    with open(fq, "w") as fh:
        for k, s in enumerate(reads):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))
    return str(fq)


def test_amplicon_count_limits(eng, tmp_path):
    """C2B_MAX_REFS = 32 amplicons run (the count sweep checks them against the oracle); 33 without a per-read ref_id are
    refused by process_fastq, process_fastq_sharded and process_bam before the FASTQ or SAM text is read, naming the limit
    and the count, with no launch; the engine refuses such a batch too."""
    engine, gpu = eng
    rng = np.random.default_rng(33)
    m = O.make_matrix()
    base, seqs, edits = allele_panel(rng, MAX_REFS + 1)
    refs, names = panel_refs(seqs)
    reads = [base, seqs[32], rc(seqs[0])]
    launch_plan = check_plan(engine, {k: refs[k] for k in names[:32]}, names[:32], reads, m)
    assert launch_plan.alns.shape[1] == MAX_REFS
    args = PU.args_from({k: getattr(O.Params(), k) for k in vars(O.Params())})
    missing = str(tmp_path / "does_not_exist.fastq")            # refused before the file is opened
    from crispresso2_b200 import bam
    before = engine.launch_count()
    for call in (lambda: core.process_fastq(missing, {}, names, refs, args, [], str(tmp_path), engine=engine, aln_matrix=m),
                 lambda: core.process_fastq_sharded(missing, {}, names, refs, args, [], str(tmp_path), engine=engine, aln_matrix=m),
                 lambda: bam.process_bam(missing, "", str(tmp_path / "o.bam"), {}, names, refs, args, [], str(tmp_path),
                                         engine=engine, aln_matrix=m)):
        with pytest.raises(EngineError) as ex:
            call()
        assert "C2B_MAX_REFS" in str(ex.value) and "33" in str(ex.value) and "32" in str(ex.value), str(ex.value)
    assert engine.launch_count() == before
    engine.configure(refs, names, m, -20, -2, 5, 2, 0, "ACGTN", 48)
    with pytest.raises(EngineError) as ex:
        engine.align(reads)
    assert "(%d)" % _lib.E_LIMIT in str(ex.value) and "C2B_MAX_REFS" in str(ex.value)
    assert engine.launch_count() == before


def test_pooled_amplicon_limit_and_winner_bit(eng):
    """Pooled runs (a per-read ref_id) configure up to C2B_MAX_POOLED_REFS = 1024 amplicons and refuse 1025; under ref_id
    the read's winner_mask carries bit ref_id mod 32 (include/c2b200.h)."""
    engine, gpu = eng
    rng = np.random.default_rng(1024)
    m = O.make_matrix()
    amps = [rand_seq(rng, 40) for _ in range(MAX_POOLED + 1)]
    refs = {"P%04d" % k: SH.shape_ref(s, seed_len=8, exclude=4) for k, s in enumerate(amps)}
    names = list(refs)
    with pytest.raises(EngineError) as ex:
        engine.configure(refs, names, m, -20, -2, 5, 2, 0, "ACGTN", 16)
    assert "(%d)" % _lib.E_LIMIT in str(ex.value) and "C2B_MAX_POOLED_REFS" in str(ex.value)
    names = names[:MAX_POOLED]
    engine.configure({k: refs[k] for k in names}, names, m, -20, -2, 5, 2, 0, "ACGTN", 16)
    picks = [0, 1, 31, 32, 33, 63, 64, 511, 512, 1000, 1022, 1023] + ([int(x) for x in rng.integers(0, MAX_POOLED, 500)] if gpu else [])
    reads = []
    for k in picks:
        s = amps[k]
        reads.append(s if len(reads) % 3 else s[:20] + ("A" if s[20] != "A" else "C") + s[21:])
    rid = np.asarray(picks, dtype=np.int32)
    engine.counts_reset()
    res = engine.align(reads, ref_id=rid)
    assert (res.recs["best_score_milli"] > 0).all()
    assert (res.recs["winner_mask"] == (np.uint32(1) << (rid % 32).astype(np.uint32))).all(), res.recs["winner_mask"]
    assert (res.recs["best_ref"] == rid).all()
    for i, k in enumerate(picks[:12]):
        nm = names[k]
        want = O.new_variant(O.Params(), reads[i], {nm: refs[nm]}, [nm], m)
        assert (res.pair(i, 0)[0], res.pair(i, 0)[1], res.score(i, 0)) == tuple(want["ref_aln_details"][0][1:]), (i, k)
