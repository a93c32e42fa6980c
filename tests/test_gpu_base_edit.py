"""--base_editor_output allele tables through the sm_90a library against the reference's own get_upset_plot_counts and
get_base_edit_dataframe_around_cut (tests/base_edit_util.py): the hand-built and failing rows, engine frames of base-editing
reads, the frames of 1 Mi synthetic reads (single amplicon and HDR), the reference's own unit tests, and one launcher-vs-CLI
run with --base_editor_output."""
import os
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import base_edit_util as U  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not U.HAVE_REF, reason="needs oracle/_ref/install")]


@pytest.fixture(scope="module")
def eng():
    from crispresso2_b200.engine import Engine
    return Engine()


def test_hand_built_and_failing_rows(eng):
    for _, df, bp, wt in U.hand_cases() + U.upset_error_cases():
        U.check_upset(df, bp, wt, eng)
        U.check_upset(df, bp, wt, eng, chunk=1)
    for _, df, nuc in U.quilt_cases() + U.quilt_error_cases():
        U.check_quilt(df, nuc, eng)
        U.check_quilt(df, nuc, eng, chunk=1)


def test_engine_frames_over_many_chunks(eng):
    rng = np.random.default_rng(41)
    fanc, fanc_hdr = U.fanc()
    g = fanc.index(U.FANC_GUIDE)
    df, names = U.engine_frame(eng, [fanc, fanc_hdr], U.base_edit_reads(rng, fanc, 3000) +
                               U.base_edit_reads(rng, fanc_hdr, 600, guide=fanc_hdr[g:g + 20]))
    bp = U.guide_targets(fanc)
    for chunk in (0, 37):
        for wt in names:
            assert U.check_upset(df, bp, wt, eng, chunk=chunk)[0] == "ok"
            assert U.check_quilt(df.loc[df["Reference_Name"] == wt], "C", eng, chunk=chunk)[0] == "ok"


@pytest.mark.parametrize("config", ["single", "hdr"])
def test_one_mebi_read_frames(eng, config):
    import base_edit_bench
    with tempfile.TemporaryDirectory() as d:
        df, bp, wt, _ = base_edit_bench.bench_frame(config, 1 << 20, d, eng)
    assert len(df) > 100000
    assert U.check_upset(df, bp, wt, eng)[0] == "ok"
    assert U.check_quilt(df.loc[df["Reference_Name"] == wt], "C", eng)[0] == "ok"


def test_reference_unit_tests_pass_against_the_drop_ins():
    import test_base_edit
    test_base_edit.run_reference_unit_tests("default")


def test_reference_cli_with_base_editor_output_is_byte_identical(tmp_path):
    import test_base_edit
    files, calls = test_base_edit.run_cli_case(tmp_path, test_base_edit.cli_cases(tmp_path)["hdr"], "default")
    assert [k for k in files if k.startswith("10i.")]
    assert calls["get_upset_plot_counts"] >= 1 and calls["get_base_edit_dataframe_around_cut"] >= 1
