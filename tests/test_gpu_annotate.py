"""--fastq_output / --bam_output annotations through the sm_90a library: the differential tests of tests/test_annotate.py on the
GPU, the shipped launcher against the unmodified CLI for both options, and a 200 k-read HDR synthetic FASTQ on which the native
writer must equal the reference's own wrappers running over the engine's lazy cache (today's launcher path)."""
import copy
import functools
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import annotate_util as AU  # noqa: E402
import test_annotate as TA  # noqa: E402
from test_cli_dropin import _snapshot  # noqa: E402

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not AU.have_reference(), reason="needs oracle/_ref/install (built by __graft_entry__.build())")]

REF_MAIN = ("import sys; sys.path.insert(0, %r); from baseline import ref_shim; CORE = ref_shim.load_core(); "
            "sys.argv = ['CRISPResso'] + sys.argv[1:]; CORE.main()" % ROOT)


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    from crispresso2_b200 import core
    tmp = tmp_path_factory.mktemp("gpu_annotate")
    old_path = os.environ["PATH"]
    os.environ["PATH"] = AU.fake_samtools(str(tmp / "bin"))
    try:
        yield TA.make_env(tmp, core.get_engine(0))            # the inputs of tests/test_annotate.py, the sm_90a engine
    finally:
        os.environ["PATH"] = old_path


def test_fanc_fixture(env):
    P = TA._pair(env, "fanc", "gpu_fanc")
    TA._check_fastq(P, env["fq"])
    TA._check_sam(P, env["fq"])


@pytest.mark.parametrize("legacy", [False, True], ids=["default", "legacy_insertions"])
def test_hdr_edges_reverse_complement_and_not_aligned(env, legacy):
    ref_names, refs, _ = env["caps"]["fanc"]
    reads = AU.edited_reads(env["fanc"], refs[ref_names[0]]["include_idxs"])
    fq = AU.write_fastq(str(env["tmp"] / ("gpu_edges_%d.fastq.gz" % legacy)), reads, gz=True)
    P = TA._pair(env, "hdr", "gpu_edges_%d" % legacy, use_legacy_insertion_quantification=legacy, expand_ambiguous_alignments=True)
    TA._check_fastq(P, fq)
    refs2 = copy.deepcopy(env["caps"]["hdr"][1])
    refs2[ref_names[0]].update(aln_chr="chr7", aln_start=1234, aln_strand="-")
    TA._check_sam(P, fq, refs=refs2)


def test_prime_editing_scaffold(env):
    TA._check_fastq(TA._pair(env, "pe", "gpu_pe"), env["pe_fq"])


@pytest.mark.parametrize("extra", [["--fastq_output"], ["--bam_output"], ["--bam_output", "--debug"]],
                         ids=["fastq_output", "bam_output", "bam_output_debug"])
def test_launcher_against_the_unmodified_cli(extra, tmp_path):
    fanc, hdr = AU.amplicons()
    fq = AU.write_fastq(str(tmp_path / "FANC.fastq"), AU.fanc_reads())
    env = dict(os.environ, PYTHONPATH=ROOT, PATH=AU.fake_samtools(str(tmp_path / "bin")))
    argv = ["-r1", fq, "-a", fanc, "-g", TA.G, "-e", hdr, "--suppress_plots", "--suppress_report", "-o", "."] + extra
    outs = []
    for mode, cmd in (("ref", [sys.executable, "-c", REF_MAIN]), ("b200", [sys.executable, "-m", "crispresso2_b200.launcher"])):
        out = str(tmp_path / mode)                           # same relative -o: the SAM header carries the command line
        os.makedirs(out)
        p = subprocess.run(cmd + argv, capture_output=True, text=True, timeout=900, env=env, cwd=out)
        assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
        outs.append(out)
    a, b = _snapshot(outs[0]), _snapshot(outs[1])
    assert sorted(a) == sorted(b)
    assert [k for k in a if a[k] != b[k]] == []
    assert any(k.endswith("CRISPResso_output.fastq.gz" if extra == ["--fastq_output"] else "CRISPResso_output.bam") for k in a)


def test_200k_hdr_reads_equal_the_reference_wrappers_over_the_lazy_cache(tmp_path):
    """the reference's process_fastq_write_out / process_single_fastq_write_bam_out with process_fastq re-bound to the engine
    (the launcher's path before the native writer) against crispresso2_b200.annotate, 200 k synthetic HDR reads"""
    import types
    import bench
    from baseline import ref_shim
    from crispresso2_b200 import annotate, core, synth
    from oracle import oracle as O
    CORE = ref_shim.load_core()
    n = int(os.environ.get("C2B_ANNOTATE_TEST_READS", "200000"))
    w = bench.Workload("hdr", n, 0)
    fq = str(tmp_path / "hdr.fastq")
    synth.write_fastq_fast(fq, w.buf.reshape(n, -1))
    args = types.SimpleNamespace(**vars(w.params))
    args.use_legacy_insertion_quantification = False
    args.prime_editing_pegRNA_scaffold_seq = args.prime_editing_pegRNA_extension_seq = ""
    args.needleman_wunsch_aln_matrix_loc = "EDNAFULL"
    args.n_processes = "1"
    args.debug = True
    refs = copy.deepcopy(w.refs)
    for nm in w.ref_names:
        refs[nm].update(aln_chr=nm, aln_start=1, aln_strand="+", sequence_length=len(refs[nm]["sequence"]))
    pf = functools.partial(core.process_fastq, engine=core.get_engine(0), aln_matrix=O.make_matrix())
    saved, old_path = CORE.process_fastq, os.environ["PATH"]
    CORE.process_fastq = pf
    os.environ["PATH"] = AU.fake_samtools(str(tmp_path / "bin"))
    try:
        outs = {}
        for tag, fn in (("ref", CORE.process_fastq_write_out),
                        ("b200", functools.partial(annotate.process_fastq_write_out, process_fastq=pf))):
            out = str(tmp_path / ("%s.fastq.gz" % tag))
            fn(fq, out, {}, w.ref_names, refs, args, [], str(tmp_path))
            with gzip.open(out, "rb") as fh:
                outs[tag] = fh.read()
        assert outs["ref"] == outs["b200"] and outs["ref"].count(b"\n") == 4 * n
        header = AU.bam_header(w.ref_names, refs)
        sams = {}
        for tag, fn in (("ref", CORE.process_single_fastq_write_bam_out),
                        ("b200", functools.partial(annotate.process_single_fastq_write_bam_out, process_fastq=pf))):
            bam = str(tmp_path / ("%s.bam" % tag))
            fn(fq, bam, header, {}, w.ref_names, refs, args, [], str(tmp_path))
            with open(bam + ".sam", "rb") as fh:
                sams[tag] = fh.read()
        assert sams["ref"] == sams["b200"] and sams["ref"].count(b"\n") == n + header.count("\n")
    finally:
        CORE.process_fastq, os.environ["PATH"] = saved, old_path
    assert np.any(np.frombuffer(outs["b200"][:1 << 20], dtype=np.uint8) == ord("&"))      # several amplicons in the annotations
