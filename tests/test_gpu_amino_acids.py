"""--coding_seq amino-acid tables through the sm_90a library against the reference's own get_amino_acid_dataframe and
global_align (tests/amino_util.py): the protein DP, the hand-built and failing rows, engine frames of coding-sequence reads, the
frames of 1 Mi synthetic reads (single amplicon and HDR) against the reference on a prefix and against the emulator build, the
reference's own unit tests, and one launcher-vs-CLI run with a coding sequence."""
import os
import sys
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import amino_util as U  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not U.HAVE_REF, reason="needs oracle/_ref/install")]


@pytest.fixture(scope="module")
def eng():
    from crispresso2_b200.engine import Engine
    return Engine()


def test_protein_dp_against_reference_global_align(eng):
    import test_amino_acids as T
    T.check_protein_dp(eng, n_random=300)
    T.check_alphabets(eng)
    T.check_overflow_refused(eng)


def test_hand_built_failing_and_refused_rows(eng):
    for label, df, left, sl, cut in U.hand_cases():
        if label.startswith("suffix_") and int(label.split("_")[1]) < 3:
            continue
        for chunk in (0, 1):
            assert U.check(df, left, sl, cut, eng, chunk=chunk)[0] == "ok"
    for _, df, left, sl, cut in U.error_cases():
        for chunk in (0, 1):
            assert U.check(df, left, sl, cut, eng, chunk=chunk)[0] != "ok"
    for _, df, left, sl, cut in U.empty_cases():
        assert "row %d" % (len(df) - 1) in U.refuses_empty(df, left, sl, cut, eng)


@pytest.mark.parametrize("hdr", [False, True])
def test_engine_frames_of_coding_reads(eng, hdr):
    import test_amino_acids as T
    T.test_engine_frames_of_coding_reads(eng, hdr)


@pytest.mark.parametrize("config", ["single", "hdr"])
def test_one_mebi_read_frames(eng, config):
    """the full frame through the drop-in; its first 50 000 rows equal the reference's frame, its first 5 000 the emulator
    build's"""
    import pandas as pd
    import amino_acid_bench
    import build_emu
    from crispresso2_b200 import amino_acids
    from crispresso2_b200.engine import Engine
    with tempfile.TemporaryDirectory() as d:
        df, left, sl, cut, _ = amino_acid_bench.bench_frame(config, 1 << 20, d, eng)
    assert len(df) > 100000
    full = amino_acids.get_amino_acid_dataframe(df, left, sl, U.reference()[2], cut, engine=eng)
    assert len(full) > 100
    prefix = df.iloc[:50000]
    assert U.check(prefix, left, sl, cut, eng)[0] == "ok"
    prefix = prefix.iloc[:5000]
    emu = amino_acids.get_amino_acid_dataframe(prefix, left, sl, U.reference()[2], cut, engine=Engine(lib_path=build_emu.build()))
    pd.testing.assert_frame_equal(amino_acids.get_amino_acid_dataframe(prefix, left, sl, U.reference()[2], cut, engine=eng), emu,
                                  check_exact=True)


def test_reference_unit_tests_pass_against_the_drop_in():
    import test_amino_acids as T
    T.run_reference_unit_tests("default")


def test_reference_cli_with_coding_seq_is_byte_identical(tmp_path):
    import test_amino_acids as T
    files, calls = T.run_cli_case(tmp_path, T.cli_cases(tmp_path)["hdr"], "default")
    assert calls["get_amino_acid_dataframe"] == len([k for k in files if "amino_acid_table_for_" in k]) >= 1
