"""--coding_seq amino-acid tables (crispresso2_b200.amino_acids, csrc/c2b_amino.cuh) on the warp-emulator build against the
reference's own get_amino_acid_dataframe and CRISPResso2Align.global_align (the package under oracle/_ref/install): the protein
DP, hand-built rows at the edges, error parity, engine frames of coding-sequence reads, the reference's own unit tests with the
drop-in standing in, and byte-identical CLI output folders.  CPU only."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)

import amino_util as U  # noqa: E402

pytestmark = pytest.mark.skipif(not U.HAVE_REF, reason="needs oracle/_ref/install (built by __graft_entry__.build())")


@pytest.fixture(scope="module")
def eng():
    import build_emu
    from crispresso2_b200.engine import Engine
    return Engine(lib_path=build_emu.build())


def _blosum():
    _, A, path = U.reference()
    return A, A.read_matrix(path)


def check_protein_dp(eng, n_random=60):
    """c2b_protein_align (batched and through align.global_align) against the reference's Cython global_align"""
    from crispresso2_b200 import align
    A, m = _blosum()
    rng = np.random.default_rng(5)
    cases = []
    for a, b in U.protein_pairs(rng, n_random):                     # random pairs of 1-341 residues, an incentive somewhere
        gi = np.zeros(len(b) + 1, dtype=int)
        gi[int(rng.integers(0, len(b) + 1))] = 1
        cases.append((a, b, gi, -1, -1))
    for k in range(5):                                             # an incentive at every position (the ATTTA / ATTA sweep)
        gi = np.zeros(5, dtype=int)
        gi[k] = 1
        cases += [("MKKKM", "MKKM", np.r_[gi[:4], 0], -1, -1), ("MKKM", "MKKKM", np.r_[gi, 0][:6], -1, -1)]
    for rep in ("KKKKKKKKKK", "KAKAKAKAKA", "WWW*WWW*WW", "**********"):    # tie-heavy repeats and stops
        cases += [(rep[:7], rep, np.zeros(11, dtype=int), -1, -1), (rep, rep[:6] + "*", np.zeros(8, dtype=int), -1, -1)]
    for go, ge in ((-5, -1), (-10, -2), (-1, -3), (0, 0), (-3, -3)):
        a, b = U.protein_pairs(rng, 1, 20, 80)[0]
        cases.append((a, b, np.zeros(len(b) + 1, dtype=int), go, ge))
    for a, b, gi, go, ge in cases:
        want = A.global_align(a, b, matrix=m, gap_incentive=gi, gap_open=go, gap_extend=ge)
        assert U.protein_batch(eng, [a], b, m, gi, go, ge)[0] == want, (a, b)
        assert align.global_align(a, b, matrix=m, gap_incentive=gi, gap_open=go, gap_extend=ge, engine=eng) == want, (a, b)
    # one batch of many reads against one reference
    b = U.protein_pairs(rng, 1, 150, 200)[0][1]
    reads = [p[0] for p in U.protein_pairs(rng, 40, 1, 170)]
    gi = np.zeros(len(b) + 1, dtype=int)
    gi[60] = 1
    assert U.protein_batch(eng, reads, b, m, gi) == [A.global_align(r, b, matrix=m, gap_incentive=gi) for r in reads]


def check_alphabets(eng):
    """read alphabets of 9, 21 and 32 symbols (a matrix over printable ASCII), and of 33 refused"""
    from crispresso2_b200 import align
    from crispresso2_b200.engine import EngineError
    A, _ = _blosum()
    rng = np.random.default_rng(9)
    syms = [chr(c) for c in range(40, 40 + 33)]
    m = rng.integers(-6, 7, size=(128, 128)).astype(np.int64)
    for nq in (9, 21, 32):
        a = "".join(syms[:nq]) + "".join(rng.choice(syms[:nq], 60))
        b = "".join(rng.choice(syms[:nq], 70))
        gi = np.zeros(len(b) + 1, dtype=int)
        gi[10] = 2
        want = A.global_align(a, b, matrix=m, gap_incentive=gi)
        assert align.global_align(a, b, matrix=m, gap_incentive=gi, engine=eng) == want
    with pytest.raises(EngineError, match="C2B_AA_MAX_Q"):
        align.global_align("".join(syms), "ABC", matrix=m, gap_incentive=np.zeros(4, dtype=int), engine=eng)


def check_overflow_refused(eng):
    """scores that can leave the DP's int32 are refused, never aligned differently"""
    from crispresso2_b200.engine import EngineError
    _, m = _blosum()
    a, b = "MKV" * 100, "MKL" * 110
    with pytest.raises(EngineError, match="int32 range"):
        U.protein_batch(eng, [a], b, m, np.zeros(len(b) + 1, dtype=int), go=-30000, ge=-1)
    big = np.asarray(m).copy()
    big[ord("M"), ord("M")] = 1 << 28
    with pytest.raises(EngineError, match="out of range"):
        U.protein_batch(eng, ["MK"], "MK", big, np.zeros(3, dtype=int))


def test_protein_dp_against_reference_global_align(eng):
    check_protein_dp(eng)
    check_alphabets(eng)
    check_overflow_refused(eng)


def test_dna_alphabets_keep_their_path(eng):
    from crispresso2_b200 import align
    _, A, _ = U.reference()
    m = A.make_matrix()
    gi = np.zeros(9, dtype=int)
    assert align.global_align("ACGTTACG", "ACGTACGT", matrix=m, gap_incentive=gi, engine=eng) == \
        A.global_align("ACGTTACG", "ACGTACGT", matrix=m, gap_incentive=gi)


@pytest.mark.parametrize("case", [c[0] for c in U.hand_cases()])
def test_hand_built_rows(eng, case):
    _, df, left, sl, cut = [c for c in U.hand_cases() if c[0] == case][0]
    if case.startswith("suffix_") and int(case.split("_")[1]) < 3:
        assert "row 0" in U.refuses_empty(df, left, sl, cut, eng)
        return
    assert U.check(df, left, sl, cut, eng)[0] == "ok"
    U.check(df, left, sl, cut, eng, chunk=1)                       # one row per device pass


@pytest.mark.parametrize("case", [c[0] for c in U.error_cases()])
def test_errors_first_failing_row_wins(eng, case):
    _, df, left, sl, cut = [c for c in U.error_cases() if c[0] == case][0]
    assert U.check(df, left, sl, cut, eng)[0] != "ok"
    U.check(df, left, sl, cut, eng, chunk=1)


def test_translation_shorter_than_a_codon_is_refused(eng):
    for _, df, left, sl, cut in U.empty_cases():
        for chunk in (0, 1):
            msg = U.refuses_empty(df, left, sl, cut, eng, chunk)
            assert "row %d" % (len(df) - 1) in msg and ("global_align is undefined" in msg or "SURVEY 3.2" in msg)


def test_unsupported_cells_name_their_column(eng):
    from crispresso2_b200 import amino_acids, vcf
    _, _, blosum = U.reference()
    for col, bad in (("Aligned_Sequence", U.AMP[:9] + "Ç" + U.AMP[10:]), ("Reference_Sequence", 5), ("#Reads", 1.5),
                     ("n_deleted", 0.5), ("ref_positions", "abc"), ("%Reads", 1)):
        df = U.frame([U.row(U.AMP)])
        df[col] = [bad]
        with pytest.raises(vcf.UnsupportedCell, match=repr(col)[1:-1]):
            amino_acids.get_amino_acid_dataframe(df, U.LEFT, 10, blosum, 1, engine=eng)


def test_timings_are_left(eng):
    from crispresso2_b200 import amino_acids
    _, df, left, sl, cut = U.hand_cases()[0]
    amino_acids.get_amino_acid_dataframe(df, left, sl, U.reference()[2], cut, engine=eng)
    t = amino_acids.get_amino_acid_dataframe.last_timings
    assert set(t) == {"pack", "rows", "align", "group", "frame", "pairs"} and t["pairs"] >= 6


def coding_reads(rng, amp, cds_start, n):
    """reads over a coding sequence: silent and missense substitutions, in-frame and frameshift indels, unedited reads"""
    out = []
    for k in range(n):
        s = list(amp)
        kind = k % 8
        p = cds_start + int(rng.integers(0, 60))
        if kind == 1:
            s[p] = "ACGT"[int(rng.integers(0, 4))]
        elif kind == 2:
            s[p] = "ACGT"[int(rng.integers(0, 4))]
            s[p + 7] = "ACGT"[int(rng.integers(0, 4))]
        elif kind == 3:
            del s[p:p + 3]
        elif kind == 4:
            del s[p:p + int(rng.integers(1, 3))]
        elif kind == 5:
            s[p:p] = list("ACGT"[int(rng.integers(0, 4))] * int(rng.integers(1, 4)))
        out.append("".join(s))
    return out


def engine_frame(eng, amps, reads):
    import base_edit_util as B
    return B.engine_frame(eng, amps, reads)


@pytest.mark.parametrize("hdr", [False, True])
def test_engine_frames_of_coding_reads(eng, hdr):
    """AlleleTable(...).to_dataframe() after process_fastq over reads with edits in a coding sequence, one and two coding
    sequences, with the HDR amplicon (-e), over several chunks"""
    import base_edit_util as B
    rng = np.random.default_rng(17 + hdr)
    fanc, fanc_hdr = B.fanc()
    amps = [fanc, fanc_hdr] if hdr else [fanc]
    reads = coding_reads(rng, fanc, 56, 300) + (coding_reads(rng, fanc_hdr, 56, 60) if hdr else [])
    df, names = engine_frame(eng, amps, reads)
    assert len(df) > 30 and df["n_inserted"].gt(0).any() and df["n_deleted"].gt(0).any()
    for nm in names:
        sub = df.loc[df["Reference_Name"] == nm]                     # as prep_amino_acid_table passes it
        for left, sl, cut in ((56, 17, 8), (100, 10, 0), (56, 50, 200)):     # two coding sequences; an out-of-range cut point
            for chunk in (0, 13):
                assert U.check(sub, left, sl, cut, eng, chunk=chunk)[0] == "ok"


def run_reference_unit_tests(lib):
    """the reference's own prep_amino_acid_table unit tests through pytest, with the drop-in standing in"""
    src = os.path.join(ROOT, "oracle", "_ref", "unit_tests", "test_data_prep.py")
    env = dict(os.environ, C2B_AMINO_LIB=lib, PYTHONPATH=os.pathsep.join([HERE, ROOT]))
    with tempfile.TemporaryDirectory() as d:
        p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "amino_acid_standin", "-p", "no:cacheprovider", "--rootdir", d,
                            src + "::TestPrepAminoAcidTable"], capture_output=True, text=True, timeout=1800, env=env, cwd=d)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-2000:]
    return p.stdout


@pytest.mark.skipif(not os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "unit_tests", "test_data_prep.py")),
                    reason="needs oracle/_ref/unit_tests")
def test_reference_unit_tests_pass_against_the_drop_in():
    import build_emu
    out = run_reference_unit_tests(build_emu.build())
    assert int(out.strip().splitlines()[-1].split(" passed")[0].split()[-1]) >= 4


CDS_FANC = "GGGCCTTCGCGCACCTCATGGAATCCCTTCTGCAGCACCTGGATCGCTTTT"


def cli_cases(tmp):
    import base_edit_util as B
    import test_cli_dropin as T
    fanc, fanc_hdr = B.fanc()
    rng = np.random.default_rng(4)
    fq = os.path.join(str(tmp), "coding.fastq")
    B.write_fastq(fq, coding_reads(rng, fanc, 56, 320))
    g = B.FANC_GUIDE
    base = ["-r1", fq, "-a", fanc, "-g", g, "-c", CDS_FANC]
    return {
        "one_coding_seq": base,
        "two_coding_seqs": base[:-1] + [CDS_FANC + "," + fanc[110:140]],
        "hdr": base + ["-e", fanc_hdr],
        "fanc_params": T._cases(tmp)["fanc_params"],
    }


def run_cli_case(tmp_path, argv, lib):
    import test_cli_dropin as T
    ref_dir, b200_dir = str(tmp_path / "ref"), str(tmp_path / "b200")
    T._run("reference", "default", ref_dir, argv)
    os.makedirs(b200_dir, exist_ok=True)
    p = subprocess.run([sys.executable, os.path.join(HERE, "amino_acid_cli_runner.py"), "b200", lib, b200_dir,
                        os.path.join(b200_dir, "_vectors.json"), "--"] + argv, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    with open(os.path.join(b200_dir, "_amino_acid_calls.json")) as fh:
        calls = json.load(fh)
    a, b = T._snapshot(ref_dir), T._snapshot(b200_dir)
    assert sorted(a) == sorted(b)
    assert not [k for k in a if a[k] != b[k]]
    return a, calls


@pytest.mark.parametrize("case", ["one_coding_seq", "two_coding_seqs", "hdr", "fanc_params"])
def test_reference_cli_with_coding_seq_is_byte_identical(case, tmp_path):
    import build_emu
    import test_cli_dropin as T
    if not T.HAVE_REF:
        pytest.skip("needs oracle/_ref/install")
    files, calls = run_cli_case(tmp_path, cli_cases(tmp_path)[case], build_emu.build())
    tables = [k for k in files if "amino_acid_table_for_" in k]
    assert tables and calls["get_amino_acid_dataframe"] == len(tables)
    if case == "two_coding_seqs":
        assert len(tables) >= 2
