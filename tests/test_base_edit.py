"""--base_editor_output allele tables (crispresso2_b200.base_edit, csrc/c2b_base_edit.cuh) on the warp-emulator build against
the reference's own get_upset_plot_counts and get_base_edit_dataframe_around_cut (the package under oracle/_ref/install):
hand-built rows, error parity, engine frames of base-editing reads, the reference's own unit tests with the drop-ins standing
in, and byte-identical CLI output folders.  CPU only."""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, HERE)

import base_edit_util as U  # noqa: E402

pytestmark = pytest.mark.skipif(not U.HAVE_REF, reason="needs oracle/_ref/install (built by __graft_entry__.build())")


@pytest.fixture(scope="module")
def eng():
    import build_emu
    from crispresso2_b200.engine import Engine
    return Engine(lib_path=build_emu.build())


@pytest.mark.parametrize("case", [c[0] for c in U.hand_cases()])
def test_upset_hand_built_rows(eng, case):
    _, df, bp, wt = [c for c in U.hand_cases() if c[0] == case][0]
    assert U.check_upset(df, bp, wt, eng)[0] == "ok"
    U.check_upset(df, bp, wt, eng, chunk=1)                      # one row per device pass


@pytest.mark.parametrize("case", [c[0] for c in U.upset_error_cases()])
def test_upset_errors_first_failing_row_wins(eng, case):
    _, df, bp, wt = [c for c in U.upset_error_cases() if c[0] == case][0]
    U.check_upset(df, bp, wt, eng)
    U.check_upset(df, bp, wt, eng, chunk=1)


@pytest.mark.parametrize("case", [c[0] for c in U.quilt_cases()])
def test_quilt_hand_built_rows(eng, case):
    _, df, nuc = [c for c in U.quilt_cases() if c[0] == case][0]
    assert U.check_quilt(df, nuc, eng)[0] == "ok"
    U.check_quilt(df, nuc, eng, chunk=1)


def test_quilt_kahan_sum_differs_from_naive(eng):
    _, df, nuc = [c for c in U.quilt_cases() if c[0] == "kahan"][0]
    want = U.check_quilt(df, nuc, eng)[1]
    assert want["%Reads"].iloc[0] != sum(df["%Reads"].tolist())


@pytest.mark.parametrize("case", [c[0] for c in U.quilt_error_cases()])
def test_quilt_errors_first_failing_row_wins(eng, case):
    _, df, nuc = [c for c in U.quilt_error_cases() if c[0] == case][0]
    U.check_quilt(df, nuc, eng)
    U.check_quilt(df, nuc, eng, chunk=1)


def test_unsupported_cells_name_their_column(eng):
    from crispresso2_b200 import base_edit, vcf
    R = U.R
    bp = [(4, "C", "T")]
    for col, bad in (("Aligned_Sequence", R[:4] + "Ç" + R[5:]), ("Reference_Sequence", 5), ("#Reads", 1.5), ("n_deleted", 0.0),
                     ("n_inserted", "1")):
        df = U.frame([U.row(R, R, 2)])
        df[col] = [bad]
        with pytest.raises(vcf.UnsupportedCell, match=repr(col)[1:-1]):
            base_edit.get_upset_plot_counts(df, bp, "A", engine=eng)
    for bad in ([(4.0, "C", "T")], [(4, "C")], [(4, "C", 5)], [(4, "C", "Ţ")], [(1 << 64, "C", "T")]):
        with pytest.raises(vcf.UnsupportedCell, match="bp_substitutions_arr"):
            base_edit.get_upset_plot_counts(U.frame([U.row(R, R, 2)]), bad, "A", engine=eng)
    df = U.frame([U.row(R, R, 2), U.row(5, None, 1, name="B")])           # other references: their cells are never read
    U.check_upset(df, bp, "A", eng)
    for col, bad in (("Aligned_Sequence", None), ("Reference_Sequence", R[:4] + "Ç" + R[5:]), ("#Reads", 2.0), ("n_mutated", 1.0),
                     ("%Reads", 1)):
        df = U.frame([U.row(R, R, 2)])
        df[col] = [bad]
        with pytest.raises(vcf.UnsupportedCell, match=repr(col)[1:-1].replace("%", "%")):
            base_edit.get_base_edit_dataframe_around_cut(df, "C", engine=eng)


def test_timings_are_left(eng):
    from crispresso2_b200 import base_edit
    _, df, bp, wt = U.hand_cases()[0]
    base_edit.get_upset_plot_counts(df, bp, wt, engine=eng)
    base_edit.get_base_edit_dataframe_around_cut(df, "C", engine=eng)
    for fn in (base_edit.get_upset_plot_counts, base_edit.get_base_edit_dataframe_around_cut):
        assert set(fn.last_timings) == {"pack", "device", "host", "frame"}
        assert all(v >= 0 for v in fn.last_timings.values())


@pytest.mark.parametrize("hdr", [False, True])
def test_engine_frames_of_base_editing_reads(eng, hdr):
    """AlleleTable(...).to_dataframe() after process_fastq over FANC.Cas9-like base-editing reads, one amplicon and with the
    HDR amplicon (-e), over several chunks"""
    rng = np.random.default_rng(31 + hdr)
    fanc, fanc_hdr = U.fanc()
    amps = [fanc, fanc_hdr] if hdr else [fanc]
    g = fanc.index(U.FANC_GUIDE)
    reads = U.base_edit_reads(rng, fanc, 300) + (U.base_edit_reads(rng, fanc_hdr, 60, guide=fanc_hdr[g:g + 20]) if hdr else [])
    df, names = U.engine_frame(eng, amps, reads)
    assert len(df) > 40 and df["n_inserted"].gt(0).any() and df["n_deleted"].gt(0).any()
    bp = U.guide_targets(fanc)
    assert len(bp) >= 5
    for chunk in (0, 7):
        for wt in names:
            want = U.check_upset(df, bp, wt, eng, chunk=chunk)
            assert want[0] == "ok" and want[1]["total_alleles_on_ref"] > 0
        assert len(U.check_upset(df, bp + [(117, "G", "-"), (0, "C", "CA")], names[0], eng, chunk=chunk)[1]["precise_allele_counts"]) > 5
        for nm in names:
            sub = df.loc[df["Reference_Name"] == nm]                 # as prep_base_edit_quilt passes it
            for nuc in ("C", "A", "G", "T"):
                assert U.check_quilt(sub, nuc, eng, chunk=chunk)[0] == "ok"


def run_reference_unit_tests(lib):
    """the reference's own base-editing unit tests through pytest, with the drop-ins standing in (tests/base_edit_standin.py);
    from a copy in a temporary directory that holds their fixture at tests/test_be_df.txt.  test_CRISPRessoCORE.py imports
    pytest_check and inline_snapshot, which are not always installed: it runs only where both import."""
    src = os.path.join(ROOT, "oracle", "_ref", "unit_tests")
    env = dict(os.environ, C2B_BASE_EDIT_LIB=lib, PYTHONPATH=os.pathsep.join([HERE, ROOT]))
    sel = ["test_data_prep.py::TestGetUpsetPlotCounts", "test_data_prep.py::TestWriteBaseEditCounts",
           "test_data_prep.py::TestPrepBaseEditQuilt"]
    have = subprocess.run([sys.executable, "-c", "import pytest_check, inline_snapshot"], capture_output=True).returncode == 0
    if have:
        sel += ["test_CRISPRessoCORE.py::test_get_upset_plot_counts", "test_CRISPRessoCORE.py::test_write_base_edit_counts"]
    with tempfile.TemporaryDirectory() as d:
        tests = os.path.join(d, "unit_tests")
        os.makedirs(tests)
        for f in {s.split("::")[0] for s in sel}:
            shutil.copy(os.path.join(src, f), tests)
        os.makedirs(os.path.join(d, "tests"))
        shutil.copy(os.path.join(HERE, "golden", "test_be_df.txt"), os.path.join(d, "tests", "test_be_df.txt"))
        p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "base_edit_standin", "-p", "no:cacheprovider", "--rootdir", d]
                           + [os.path.join(tests, s) for s in sel], capture_output=True, text=True, timeout=1800, env=env, cwd=d)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-2000:]
    assert " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-2000:]
    return p.stdout


@pytest.mark.skipif(not os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "unit_tests", "test_data_prep.py")),
                    reason="needs oracle/_ref/unit_tests")
def test_reference_unit_tests_pass_against_the_drop_ins():
    import build_emu
    out = run_reference_unit_tests(build_emu.build())
    assert int(out.strip().splitlines()[-1].split(" passed")[0].split()[-1]) >= 4


def cli_cases(tmp):
    """--base_editor_output (no -qwc, so that the 10i tables are written) on base-editing reads of the FANC amplicon"""
    fanc, fanc_hdr = U.fanc()
    rng = np.random.default_rng(3)
    fq = os.path.join(str(tmp), "base_edit.fastq")
    reads = U.base_edit_reads(rng, fanc, 240) + U.base_edit_reads(rng, fanc, 60, nuc_from="A", nuc_to="G")
    U.write_fastq(fq, reads)
    g = U.FANC_GUIDE
    base = ["-r1", fq, "-a", fanc, "-g", g, "--base_editor_output"]
    return {
        "default": base,
        "two_guides": base[:-2] + [g + "," + fanc[150:170], "--base_editor_output"],
        "a_to_g": base + ["--conversion_nuc_from", "A", "--conversion_nuc_to", "G"],
        "outside_qw": base + ["--base_editor_consider_changes_outside_qw"],
        "skip_allele": base + ["--base_editor_target_ref_skip_allele_count", "1"],
        "hdr": base + ["-e", fanc_hdr],
    }


def run_cli_case(tmp_path, argv, lib):
    import test_cli_dropin as T
    ref_dir, b200_dir = str(tmp_path / "ref"), str(tmp_path / "b200")
    T._run("reference", "default", ref_dir, argv)
    os.makedirs(b200_dir, exist_ok=True)
    p = subprocess.run([sys.executable, os.path.join(HERE, "base_edit_cli_runner.py"), "b200", lib, b200_dir,
                        os.path.join(b200_dir, "_vectors.json"), "--"] + argv, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    with open(os.path.join(b200_dir, "_base_edit_calls.json")) as fh:
        calls = json.load(fh)
    a, b = T._snapshot(ref_dir), T._snapshot(b200_dir)
    assert sorted(a) == sorted(b)
    assert not [k for k in a if a[k] != b[k]]
    return a, calls


@pytest.mark.parametrize("case", ["default", "two_guides", "a_to_g", "outside_qw", "skip_allele", "hdr"])
def test_reference_cli_with_base_editor_output_is_byte_identical(case, tmp_path):
    import build_emu
    import test_cli_dropin as T
    if not T.HAVE_REF:
        pytest.skip("needs oracle/_ref/install")
    argv = cli_cases(tmp_path)[case]
    files, calls = run_cli_case(tmp_path, argv, build_emu.build())
    assert [k for k in files if k.startswith("10i.") and k.endswith(".binary_allele_counts.txt")]
    assert [k for k in files if "base_edit_" in k and k.endswith("s_quilt.txt")]
    assert calls["get_upset_plot_counts"] >= (2 if case == "two_guides" else 1)
    assert calls["get_base_edit_dataframe_around_cut"] >= 1


def test_fanc_params_runs_the_quilt_drop_in(tmp_path):
    """the existing fanc_params CLI case (--base_editor_output with -qwc: no 10i tables) through the quilt drop-in"""
    import build_emu
    import test_cli_dropin as T
    if not T.HAVE_REF:
        pytest.skip("needs oracle/_ref/install")
    files, calls = run_cli_case(tmp_path, T._cases(tmp_path)["fanc_params"], build_emu.build())
    assert [k for k in files if "base_edit_" in k and k.endswith("s_quilt.txt")]
    assert calls["get_base_edit_dataframe_around_cut"] >= 1
