"""--vcf_output edit counts (crispresso2_b200.vcf.build_edit_counts, csrc/c2b_vcf.cuh) on the warp-emulator build against the
reference's own build_edit_counts (writers/vcf.py:172-212 of the package under oracle/_ref/install): the same dict in the same
key order, or the same exception for the same first failing row.  CPU only."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)

import vcf_util as V  # noqa: E402

pytestmark = pytest.mark.skipif(not V.HAVE_REF, reason="needs oracle/_ref/install (built by __graft_entry__.build())")


@pytest.fixture(scope="module")
def eng():
    import build_emu
    from crispresso2_b200.engine import Engine
    return Engine(lib_path=build_emu.build())


@pytest.mark.parametrize("case", [c[0] for c in V.hand_frames()])
def test_hand_built_rows(eng, case):
    _, df, amp = [c for c in V.hand_frames() if c[0] == case][0]
    V.check(df, amp, eng)
    V.check(df, amp, eng, chunk=1)                               # one row per device pass


@pytest.mark.parametrize("case", [c[0] for c in V.error_frames()])
def test_errors_first_failing_row_wins(eng, case):
    _, df, amp = [c for c in V.error_frames() if c[0] == case][0]
    want = V.check(df, amp, eng)
    assert want[0] != "ok"
    V.check(df, amp, eng, chunk=1)                               # the failing row in a later chunk than a clean one


def test_engine_frames_on_repeat_rich_amplicons(eng):
    """homopolymer, di- and trinucleotide runs at the cut: normalisation walks many steps (down to position 0 in the hand-built
    rows del_at_0 / del_whole: the aligner turns deletions at an amplicon end into end gaps)"""
    rng = np.random.default_rng(5)
    amp = V.repeat_amplicon(rng)
    df, names = V.engine_frame(eng, [amp], V.edited_reads(rng, amp, 180))
    assert len(df) > 60
    out = V.check(df, {names[0]: ("chr2", 1000)}, eng)[1]
    assert any(len(r) > 1 for (_, _, r, _) in out) and any(len(a) > 1 for (_, _, _, a) in out)
    walked = V.reference_vcf()._left_normalize_deletion
    del_rows = [r for _, r in df.iterrows() if r["deletion_coordinates"]]
    assert max(s - walked(s, e, r["ref_positions"], r["Reference_Sequence"])[0] for r in del_rows for (s, e) in r["deletion_coordinates"]) >= 4
    V.check(df, {names[0]: ("chr2", 1000)}, eng, chunk=7)           # several chunks


def test_engine_frames_two_amplicons(eng):
    """two amplicons on one chrom (their counts merge) and on two; expanded ambiguous rows and AMBIGUOUS_ rows"""
    rng = np.random.default_rng(11)
    a = V.repeat_amplicon(rng)
    b = a[:200] + "".join("ACGT"[(("ACGT".index(c)) + 1) % 4] for c in a[200:])
    df, names = V.engine_frame(eng, [a, b], V.edited_reads(rng, a, 96) + V.edited_reads(rng, b, 96))
    ok = df[~df["Reference_Name"].str.startswith("AMBIGUOUS_")].reset_index(drop=True)
    V.check(ok, {names[0]: ("7", 100), names[1]: ("7", 100)}, eng)
    V.check(ok, {names[0]: ("7", 100), names[1]: ("chrX", 1 << 40)}, eng, chunk=5)
    V.check(df, {names[0]: ("7", 100), names[1]: ("7", 100)}, eng)   # raises KeyError at the first AMBIGUOUS_ row if any


def test_unsupported_cells_name_their_column(eng):
    from crispresso2_b200 import vcf
    R = "ACGTTGCAAGGCTTAC"
    amp = {"A": ("chr1", 100)}
    for col, bad in (("Aligned_Sequence", "ACGTTGCAAGGCTTAÇ"), ("#Reads", 1.5), ("ref_positions", [0.0] * 16),
                     ("substitution_positions", "5"), ("deletion_coordinates", [(1, 2, 3)]), ("insertion_coordinates", [5]),
                     ("ref_positions", [1 << 63] * 16), ("substitution_positions", [1 << 62])):
        df = V.frame([V.row(R, R[:5] + "A" + R[6:], subs=[5])])
        df[col] = [bad]
        with pytest.raises(vcf.UnsupportedCell, match=repr(col)[1:-1]):
            vcf.build_edit_counts(df, amp, engine=eng)
    with pytest.raises(vcf.UnsupportedCell, match="amplicon_positions"):
        vcf.build_edit_counts(V.frame([V.row(R, R[:5] + "A" + R[6:], subs=[5])]), {"A": ("chr1", 1 << 62)}, engine=eng)


def test_unedited_frame_is_empty(eng):
    from crispresso2_b200 import vcf
    R = "ACGTTGCAAGGCTTAC"
    df = V.frame([V.row(R, R, n=(0, 0, 0), name="nowhere")])
    assert vcf.build_edit_counts(df, {}, engine=eng) == V.reference_vcf().build_edit_counts(df, {}) == {}


def run_reference_unit_tests(lib):
    """the reference's own tests/unit_tests/test_writers/test_vcf/*.py through pytest, with the drop-in standing in; from a copy
    in a temporary directory, because two of them write their output file next to themselves"""
    import shutil
    import tempfile
    src = os.path.join(ROOT, "oracle", "_ref", "unit_tests", "test_writers", "test_vcf")
    env = dict(os.environ, C2B_VCF_LIB=lib, PYTHONPATH=os.pathsep.join([HERE, ROOT]))
    with tempfile.TemporaryDirectory() as d:
        tests = os.path.join(d, "test_vcf")
        shutil.copytree(src, tests, ignore=shutil.ignore_patterns("__pycache__"))
        p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "vcf_standin", "-p", "no:cacheprovider", "--rootdir", d, tests],
                           capture_output=True, text=True, timeout=1800, env=env, cwd=d)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-2000:]
    return p.stdout


@pytest.mark.skipif(not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "unit_tests", "test_writers", "test_vcf")),
                    reason="needs oracle/_ref/unit_tests")
def test_reference_unit_tests_pass_against_the_drop_in():
    import build_emu
    out = run_reference_unit_tests(build_emu.build())
    assert int(out.strip().splitlines()[-1].split(" passed")[0].split()[-1]) >= 40


def cli_cases(tmp):
    """--vcf_output on FANC.Cas9 and on the HDR golden set, coordinates on one chrom and on two"""
    import test_cli_dropin as T
    base = T._cases(tmp)
    fanc = base["fanc_default"]
    return {
        "fanc_vcf": fanc + ["--vcf_output", "--amplicon_coordinates", "chr11:5000"],
        "fanc_hdr_vcf_one_chrom": base["fanc_fastq_output"][:-1] + ["--vcf_output", "--amplicon_coordinates", "chr11:5000,chr11:5000"],
        "fanc_hdr_vcf_two_chroms": base["fanc_fastq_output"][:-1] + ["--vcf_output", "--amplicon_coordinates", "7:1,chrX:1099511627776"],
    }


@pytest.mark.parametrize("case", ["fanc_vcf", "fanc_hdr_vcf_one_chrom", "fanc_hdr_vcf_two_chroms"])
def test_reference_cli_with_vcf_output_is_byte_identical(case, tmp_path):
    import build_emu
    import test_cli_dropin as T
    if not T.HAVE_REF:
        pytest.skip("needs oracle/_ref/install")
    argv = cli_cases(tmp_path)[case]
    ref_dir, b200_dir = str(tmp_path / "ref"), str(tmp_path / "b200")
    T._run("reference", "default", ref_dir, argv)
    T._run("b200", build_emu.build(), b200_dir, argv)
    a, b = T._snapshot(ref_dir), T._snapshot(b200_dir)
    assert "CRISPResso_output.vcf" in a
    assert sorted(a) == sorted(b)
    assert not [k for k in a if a[k] != b[k]]
