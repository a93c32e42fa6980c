"""Pins the CPU oracle (oracle/) against the reference: restated known-answer tests, golden vectors produced
by the compiled reference (tests/golden/gen_golden.py), and fuzzing against the compiled reference's recorded answers."""
import gzip
import json
import os
import random

import numpy as np
import pytest

from oracle import oracle as O
import golden_util as G
import reference_record


def Z(n):
    return np.zeros(n, dtype=np.int64)


# ---- known answers restated from /root/reference/tests/unit_tests/test_CRISPResso2Align.py --------------
def test_kat_identity(ednafull):
    assert O.global_align("ATTA", "ATTA", ednafull, Z(5)) == ("ATTA", "ATTA", 100.0)           # :35-40


def test_kat_gap_incentive_sweep(ednafull):                                                  # :139-273
    want = {0: ("ATT-A", "ATTTA"), 1: ("A-TTA", "ATTTA"), 2: ("AT-TA", "ATTTA"), 3: ("ATT-A", "ATTTA"),
            4: ("ATT-A", "ATTTA")}
    for pos in range(5):
        gi = Z(6)
        gi[pos] = 1
        s1, s2, sc = O.global_align("ATTA", "ATTTA", ednafull, gi)
        assert sc == 80.0 and s2 == "ATTTA" and s1.replace("-", "") == "ATTA"
        if pos in (1, 2):
            assert (s1, s2) == want[pos]


def test_kat_n_and_mismatch(ednafull):
    assert O.global_align("ANNG", "ATCG", ednafull, Z(5)) == ("A-NNG", "ATC-G", 40.0)          # :292-300
    assert O.global_align("AAAA", "TTTT", ednafull, Z(5)) == ("---AAAA", "TTTT---", 0.0)      # :324-332
    assert O.global_align("A", "A", ednafull, Z(2)) == ("A", "A", 100.0)                       # :281-289


# ---- known answers restated from test_CRISPRessoCOREResources.py ---------------------------------------
def test_kat_deletions():
    p = O.find_indels_substitutions("-ATTA", "AATTA", [1, 2, 3])                              # :11-17 (shape)
    assert p["all_deletion_positions"] == [0] and p["all_deletion_coordinates"] == [(0, 1)]
    p = O.find_indels_substitutions("AT-TA", "ATTTA", [1, 2])
    assert p["deletion_positions"] == [2] and p["deletion_n"] == 1 and p["ref_positions"] == [0, 1, 2, 3, 4]
    p = O.find_indels_substitutions("ATTT-", "ATTTA", [4])                                     # trailing deletion
    assert p["all_deletion_coordinates"] == [(4, 5)] and p["deletion_sizes"] == [1]


def test_kat_insertions():
    p = O.find_indels_substitutions("ATGGTA", "AT--TA", [1, 2])
    assert p["all_insertion_positions"] == [1, 2] and p["insertion_sizes"] == [2] and p["insertion_n"] == 2
    assert p["ref_positions"] == [0, 1, -2, -2, 2, 3]
    p = O.find_indels_substitutions("GGATTA", "--ATTA", [0, 1])                                # leading: ignored
    assert p["all_insertion_positions"] == [] and p["ref_positions"][:2] == [-1, -1]
    p = O.find_indels_substitutions("ATTAGG", "ATTA--", [2, 3])                                # trailing: ignored
    assert p["all_insertion_positions"] == []


# ---- golden vectors from the compiled reference -----------------------------------------------------------
def test_align_vectors(ednafull):
    with gzip.open(os.path.join(G.GOLD, "align_vectors.json.gz"), "rt") as fh:
        cases = json.load(fh)
    assert len(cases) >= 200
    for c in cases:
        got = O.global_align(c["read"], c["ref"], ednafull, np.array(c["gi"], dtype=np.int64), c["go"], c["ge"])
        assert got == (c["s1"], c["s2"], c["score"]), c
        p = O.find_indels_substitutions(c["s1"], c["s2"], c["inc"])
        assert not G.payload_equal(c["payload"], p), (c, p)


@pytest.mark.parametrize("case", G.CASES)
def test_whole_path_golden(case, ednafull):
    rec = G.load(case)
    refs = G.refs_from(rec)
    params = O.Params(**rec["params"])
    cache, stats, lost = O.process_reads(rec["reads"], refs, rec["ref_names"], params, ednafull)
    assert stats == rec["aln_stats"]
    assert list(cache.keys()) == list(rec["variants"].keys())
    assert set(lost) == set(rec["not_aligned"])
    for s, want in rec["variants"].items():
        got = cache[s]
        for k in ("count", "aln_ref_names", "aln_scores", "best_match_score", "class_name", "best_match_name"):
            assert got[k] == want[k], (s, k)
        assert [list(d) for d in got["ref_aln_details"]] == want["ref_aln_details"]
        for r in want["aln_ref_names"]:
            bad = G.payload_equal(want["variant_" + r], got["variant_" + r])
            assert not bad, (s, r, bad)
    names = list(rec["ref_names"])
    if rec["params"].get("prime_editing_pegRNA_scaffold_seq"):          # the reference main() appends after process_fastq (:3759-3764)
        names.append("Scaffold-incorporated")
        refs["Scaffold-incorporated"] = dict(refs["Prime-edited"])
        assert any(v["class_name"] == "Scaffold-incorporated" for v in cache.values())
    vec, sca, classes, total = O.count_vectors(cache, refs, names, params)
    for r in names:
        seq = refs[r]["sequence"]
        assert G.mod_count_text(seq, vec[r], sca[r]["counts_total"]) == G.file_for(rec, r, "Modification_count_vectors.txt")
        assert G.qw_count_text(seq, vec[r], sca[r]["counts_total"]) == G.file_for(
            rec, r, "Quantification_window_modification_count_vectors.txt")
        nf = G.nuc_freq_rows(G.file_for(rec, r, "Nucleotide_frequency_table.txt"))
        for b in "ACGTN-":
            assert (nf[b] == vec[r]["all_base_count_" + b]).all(), (r, b)


# ---- fuzz against the compiled reference (its answers recorded: tests/reference_record.py) -------------------
REC = reference_record.Record("reference_oracle_fuzz")
SREC = reference_record.Record("reference_scoring_fuzz")
MATRIX_FILE = os.path.join(G.GOLD, "scoring_nuc.matrix")


@pytest.fixture(scope="module", autouse=True)
def _save_records():
    yield
    REC.save()
    SREC.save()


def test_live_fuzz_against_compiled_reference(ednafull):
    mods = O.ref_modules() if reference_record.RECORDING else None
    rng = random.Random(7)
    m = np.ascontiguousarray(ednafull)
    for _ in range(400):
        I = rng.choice([4, 9, 30, 77, 150])
        ref = "".join(rng.choice("ACGT") for _ in range(I))
        read = "".join(c if rng.random() > 0.08 else rng.choice("ACGTN") for c in ref)
        cut = rng.randrange(I)
        read = read[:cut] + read[cut + rng.randrange(0, 6):] if rng.random() < 0.5 else read[:cut] + "ACG" + read[cut:]
        if len(read) < 3:
            continue
        gi = Z(I + 1)
        gi[rng.randrange(I + 1)] = 1
        go, ge = rng.choice([(-20, -2), (-1, -1), (-7, -3)])
        key = "align %d" % _
        want = REC.value(key, lambda: tuple(mods[0].global_align(read, ref, matrix=m, gap_incentive=gi, gap_open=go, gap_extend=ge)))
        assert O.global_align(read, ref, m, gi, go, ge) == want
        inc = sorted(rng.sample(range(I), min(I, 3)))
        w = REC.value("payload %d" % _, lambda: {k: (v.tolist() if hasattr(v, "tolist") else v)
                                                   for k, v in mods[1].find_indels_substitutions(want[0], want[1], inc).__dict__.items()})
        g = O.find_indels_substitutions(want[0], want[1], inc)
        assert not G.payload_equal(w, g)


def test_matrix_file_against_compiled_reference():
    """The NCBI-format fixture tests/golden/scoring_nuc.matrix (asymmetric, N-N above every match) read by oracle.read_matrix
    and by the reference's own read_matrix."""
    mods = O.ref_modules() if reference_record.RECORDING else None
    want = SREC.value("read_matrix", lambda: np.asarray(mods[0].read_matrix(MATRIX_FILE)))
    got = O.read_matrix(MATRIX_FILE)
    assert got.shape == want.shape and (got == want).all()
    assert got[ord("A"), ord("C")] != got[ord("C"), ord("A")] and got[ord("N"), ord("N")] > got[ord("G"), ord("G")]


def scoring_case(rng, k, ednafull):
    """Case k of the scoring-space fuzz -> (read, ref, matrix, gap_incentive, gap_open, gap_extend, label).  Matrices: make_matrix
    with varied scores (mismatch >= 0 and N-N above the match score included), asymmetric tables, the NCBI-format fixture, and
    EDNAFULL scaled by 2^16 .. 2^21 (I, J <= 150, where the reference's int32 DP is still exact).  Gap pairs include go == ge,
    go > ge, ge = 0, go = ge = 0 and positive values (only the drop-in global_align receives those).  Incentives: zero,
    cut-only, non-zero gi[0] and gi[I], dense random and negative."""
    kind = k % 5
    if kind == 0:
        m = O.make_matrix(rng.randint(1, 12), rng.randint(-12, 2), rng.randint(-6, 3), rng.randint(-3, 14))
    elif kind == 1:
        m = np.array(ednafull, dtype=np.int64)
        for a in "ACGTN":
            for b in "ACGTN":
                if rng.random() < 0.4:
                    m[ord(a), ord(b)] += rng.randint(-4, 4)
    elif kind == 2:
        m = O.read_matrix(MATRIX_FILE)
    elif kind == 3:
        m = np.array(ednafull, dtype=np.int64) << rng.randint(16, 21)
    else:
        m = np.array(ednafull, dtype=np.int64)
    I = rng.choice([5, 12, 40, 90, 150])
    ref = "".join(rng.choice("ACGT" if rng.random() < 0.8 else "ACGTN") for _ in range(I))
    read = "".join(c if rng.random() > 0.1 else rng.choice("ACGTN") for c in ref)
    cut = rng.randrange(I)
    u = rng.random()
    if u < 0.4:
        read = read[:cut] + read[cut + rng.randrange(1, 8):]
    elif u < 0.7:
        read = read[:cut] + "".join(rng.choice("ACGT") for _ in range(rng.randrange(1, 8))) + read[cut:]
    read = read[:150] or "A"
    go, ge = rng.choice([(-20, -2), (-5, -5), (-1, -5), (-10, 0), (-3, -1), (0, 0), (2, 1), (-2, 3)])
    gi = Z(I + 1)
    prof = rng.randrange(5)
    if prof == 1:
        gi[cut + 1] = rng.randint(1, 6)
    elif prof == 2:
        gi[0], gi[I], gi[cut + 1] = rng.randint(1, 5), rng.randint(1, 5), 1
    elif prof == 3:
        gi[:] = [rng.randint(0, 3) for _ in range(I + 1)]
    elif prof == 4:
        gi[cut + 1] = -rng.randint(1, 6)
        gi[rng.randrange(I + 1)] -= rng.randint(0, 3)
    if kind == 3 and rng.random() < 0.5:
        gi *= 1 << rng.randint(10, 18)
    return read, ref, np.ascontiguousarray(m), gi, go, ge, "m%d gi%d" % (kind, prof)


def test_scoring_fuzz_against_compiled_reference(ednafull):
    """The oracle beyond EDNAFULL: global_align and find_indels_substitutions of the compiled reference (answers recorded in
    tests/golden/reference_scoring_fuzz.json.gz) over matrices, gap pairs, incentive profiles and magnitudes.  Cases where
    the reference's traceback reads a pointer it never set (the oracle's rc = -3) are recorded as such."""
    mods = O.ref_modules() if reference_record.RECORDING else None
    rng = random.Random(11)
    undefined, kinds = 0, set()
    for k in range(360):
        read, ref, m, gi, go, ge, label = scoring_case(rng, k, ednafull)
        try:
            got = O.global_align(read, ref, m, gi, go, ge)
        except O.OracleUndefined:
            got = "undefined"
        want = SREC.value("align %d" % k, lambda: "undefined" if got == "undefined" else
                          tuple(mods[0].global_align(read, ref, matrix=m, gap_incentive=gi, gap_open=go, gap_extend=ge)))
        assert got == want, (k, label, go, ge)
        if got == "undefined":
            undefined += 1
            continue
        kinds.add(label)
        inc = sorted(rng.sample(range(len(ref)), min(len(ref), 4)))
        w = SREC.value("payload %d" % k, lambda: {key: (v.tolist() if hasattr(v, "tolist") else v)
                                                  for key, v in mods[1].find_indels_substitutions(want[0], want[1], inc).__dict__.items()})
        assert not G.payload_equal(w, O.find_indels_substitutions(want[0], want[1], inc)), (k, label)
    assert len(kinds) == 25 and undefined < 60, (sorted(kinds), undefined)


def test_legacy_classification_restatement_against_compiled_reference():
    """oracle.find_indels_substitutions_legacy (checker for a future device path) == the reference's compiled function on real
    alignments (random reads aligned by the reference's own global_align; its answers recorded)."""
    mods = O.ref_modules() if reference_record.RECORDING else None
    import random
    rng = random.Random(5)
    n = 0
    for _ in range(400):
        I = rng.choice([20, 41, 80, 150])
        ref = "".join(rng.choice("ACGT") for _ in range(I))
        read = list(ref)
        for _k in range(rng.randrange(0, 4)):
            p = rng.randrange(len(read))
            u = rng.random()
            if u < 0.4:
                del read[p:p + rng.randrange(1, 9)]
            elif u < 0.7:
                read[p:p] = [rng.choice("ACGT") for _q in range(rng.randrange(1, 7))]
            else:
                read[p] = rng.choice("ACGTN")
        read = "".join(read)
        if len(read) < 3:
            continue
        gi = np.zeros(I + 1, dtype=np.int64)
        gi[rng.randrange(I + 1)] = 1
        inc = sorted(rng.sample(range(I), rng.randrange(0, min(I, 10))))

        def run():
            a1, a2, _ = mods[0].global_align(read, ref, matrix=mods[0].make_matrix(), gap_incentive=gi, gap_open=-20, gap_extend=-2)
            return a1, a2, mods[1].find_indels_substitutions_legacy(a1, a2, inc)
        s1, s2, want = REC.value("legacy %d" % _, run)
        got = O.find_indels_substitutions_legacy(s1, s2, inc)
        for k, v in want.items():
            g = got[k]
            if isinstance(v, np.ndarray):
                assert list(v) == list(g), (k, s1, s2)
            else:
                assert v == g and type(v) is type(g), (k, v, g, s1, s2)
        n += 1
    assert n > 300
