"""--vcf_output edit counts through the sm_90a library against the reference's own build_edit_counts (tests/vcf_util.py): the
hand-built and failing rows, engine frames over many chunks and larger than one default chunk, the frames of 1 Mi synthetic
reads (single amplicon and HDR), the reference's own unit tests, and one launcher-vs-CLI run with --vcf_output."""
import os
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import vcf_util as V  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not V.HAVE_REF, reason="needs oracle/_ref/install")]


@pytest.fixture(scope="module")
def eng():
    from crispresso2_b200.engine import Engine
    return Engine()


def test_hand_built_and_failing_rows(eng):
    for _, df, amp in V.hand_frames() + V.error_frames():
        V.check(df, amp, eng)
        V.check(df, amp, eng, chunk=1)


def test_engine_frames_over_many_chunks(eng):
    rng = np.random.default_rng(23)
    df, amp = V.big_frame(eng, rng, 40000)                       # more rows than one default chunk (16384)
    V.check(df, amp, eng)
    V.check(df, amp, eng, chunk=997)
    a = V.repeat_amplicon(rng)
    b = a[:200] + "".join("ACGT"[(("ACGT".index(c)) + 1) % 4] for c in a[200:])
    df, names = V.engine_frame(eng, [a, b], V.edited_reads(rng, a, 2000) + V.edited_reads(rng, b, 2000))
    for amp in ({names[0]: ("7", 100), names[1]: ("7", 100)}, {names[0]: ("07", 0), names[1]: ("chrX", 1 << 40)}):
        V.check(df, amp, eng, chunk=301)


@pytest.mark.parametrize("config", ["single", "hdr"])
def test_one_mebi_read_frames(eng, config):
    import vcf_bench
    with tempfile.TemporaryDirectory() as d:
        df, amp, _ = vcf_bench.bench_frame(config, 1 << 20, d, eng, amplicon_rows_only=False)
    assert len(df) > 100000
    V.check(df, amp, eng)                                        # HDR: edited AMBIGUOUS_ rows, the KeyError of the reference CLI
    df = df[df["Reference_Name"].isin(list(amp))].reset_index(drop=True)
    want = V.check(df, amp, eng)
    assert want[0] == "ok" and len(want[1]) > 1000


def test_reference_unit_tests_pass_against_the_drop_in():
    import test_vcf
    test_vcf.run_reference_unit_tests("default")


def test_reference_cli_with_vcf_output_is_byte_identical(tmp_path):
    import test_cli_dropin as T
    import test_vcf
    argv = test_vcf.cli_cases(tmp_path)["fanc_hdr_vcf_two_chroms"]
    ref_dir, b200_dir = str(tmp_path / "ref"), str(tmp_path / "b200")
    T._run("reference", "default", ref_dir, argv)
    T._run("b200", "default", b200_dir, argv)
    a, b = T._snapshot(ref_dir), T._snapshot(b200_dir)
    assert "CRISPResso_output.vcf" in a
    assert sorted(a) == sorted(b)
    assert not [k for k in a if a[k] != b[k]]
