"""--fastq_output / --bam_output annotations (crispresso2_b200.annotate: device pass on the warp-emulator build, native writers)
against the reference's own process_fastq_write_out / process_single_fastq_write_bam_out with its own process_fastq, on the same
inputs: decompressed FASTQ bytes and SAM text identical, every cache entry equal to the reference's dict once materialised
(incl. the new key and its position), no entry materialised by the write.  CPU; needs oracle/_ref/install."""
import copy
import gzip
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))

import annotate_util as AU  # noqa: E402

pytestmark = pytest.mark.skipif(not AU.have_reference(), reason="needs oracle/_ref/install (built by __graft_entry__.build())")

G = "GGAATCCCTTCTGCAGCACC"


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    import build_emu
    from crispresso2_b200.engine import Engine
    tmp = tmp_path_factory.mktemp("annotate")
    old_path = os.environ["PATH"]
    os.environ["PATH"] = AU.fake_samtools(str(tmp / "bin"))
    try:
        yield make_env(tmp, Engine(lib_path=build_emu.build()))
    finally:
        os.environ["PATH"] = old_path


def make_env(tmp, engine):
    """inputs captured from the reference's main(): FANC alone, FANC + HDR amplicon, prime editing with a scaffold"""
    from baseline import ref_shim
    fanc, hdr = AU.amplicons()
    fq = AU.write_fastq(str(tmp / "FANC.fastq"), AU.fanc_reads())
    caps = {"fanc": AU.capture(tmp, ["-r1", fq, "-a", fanc, "-g", G]),
            "hdr": AU.capture(tmp, ["-r1", fq, "-a", fanc, "-g", G, "-e", hdr])}
    import pe_case
    pe_fq = str(tmp / "pe_scaffold.fastq")
    ext, scaffold = pe_case.write_fastq(pe_fq, fanc)
    caps["pe"] = AU.capture(tmp, ["-r1", pe_fq, "-a", fanc, "--prime_editing_pegRNA_spacer_seq", G, "--prime_editing_pegRNA_extension_seq",
                                  ext, "--prime_editing_pegRNA_scaffold_seq", scaffold])
    return {"CORE": ref_shim.load_core(), "engine": engine, "tmp": tmp, "caps": caps, "fq": fq, "pe_fq": pe_fq, "fanc": fanc}


def _pair(env, which, sub, **flags):
    ref_names, refs, args = env["caps"][which]
    args = copy.copy(args)
    for k, v in flags.items():
        setattr(args, k, v)
    d = env["tmp"] / sub
    d.mkdir(exist_ok=True)
    return AU.Pair(env["CORE"], env["engine"], d, ref_names, refs, args)


def _check_fastq(P, fq, tag="f", empty=False):
    res_r, res_b, cache_r, cache_b, text_r, text_b, untouched = P.fastq(fq, tag)
    assert untouched                                          # the write materialised no entry
    assert text_r == text_b
    assert text_r.count(b"\n") >= 4 or (empty and text_r == b"")
    AU.check_results(res_r, res_b, cache_r, cache_b)
    for v in cache_r.values():
        assert list(v.keys())[-1] == "crispresso2_annotation"


def _check_sam(P, fq, tag="s", refs=None, debug=True):
    res_r, res_b, cache_r, cache_b, sam_r, sam_b = P.sam(fq, tag, refs=refs, debug=debug)
    assert sam_r == sam_b
    AU.check_results(res_r, res_b, cache_r, cache_b)


def test_fanc_fixture_fastq_and_sam(env):
    P = _pair(env, "fanc", "fanc")
    _check_fastq(P, env["fq"])
    _check_sam(P, env["fq"])


@pytest.mark.parametrize("flags", [{}, {"expand_ambiguous_alignments": True}, {"assign_ambiguous_alignments_to_first_reference": True}],
                         ids=["default", "expand", "assign_first"])
def test_fanc_hdr(env, flags):
    P = _pair(env, "hdr", "hdr_" + "_".join(flags) or "hdr", **flags)
    _check_fastq(P, env["fq"])
    _check_sam(P, env["fq"])


@pytest.mark.parametrize("legacy", [False, True], ids=["default", "legacy_insertions"])
def test_edges_reverse_complement_and_not_aligned(env, legacy):
    ref_names, refs, _ = env["caps"]["fanc"]
    reads = AU.edited_reads(env["fanc"], refs[ref_names[0]]["include_idxs"])
    fq = AU.write_fastq(str(env["tmp"] / ("edges_%d.fastq" % legacy)), reads)
    P = _pair(env, "hdr", "edges_%d" % legacy, use_legacy_insertion_quantification=legacy, expand_ambiguous_alignments=True)
    _check_fastq(P, fq)
    _check_sam(P, fq)


def test_prime_editing_scaffold(env):
    P = _pair(env, "pe", "pe")
    _check_fastq(P, env["pe_fq"])


def _adversarial(reads):
    a, b, c = reads[:3]
    q = lambda s: "I" * len(s)
    return {
        "crlf": "@a\r\n%s\r\n+\r\n%s\r\n@b\r\n%s\r\n+\r\n%s\r\n" % (a, q(a), a, q(a)),
        "lone_cr": "@a\r%s\r+\r%s\r@b\r%s\r+\r%s\r" % (a, q(a), b, q(b)),
        "mixed_ends": "@a\n%s\r\n+\r%s\n@b\r\n%s\n+\n%s\r" % (a, q(a), a, q(a)),
        "blank_plus_and_quality": "@a\n%s\n\n\n@b\n%s\n+\n%s\n" % (a, b, q(b)),
        "whitespace": "@a \n  %s \t\n+ x \n%s  \n" % (c, q(c)),
        "no_final_newline": "@a\n%s\n+\n%s\n@b\n%s\n+\n%s" % (a, q(a), b, q(b)),
        "truncated_record": "@a\n%s\n+\n%s\n@b\n%s\n" % (a, q(a), c),
        "empty": "",
    }


@pytest.mark.parametrize("gz", [False, True], ids=["plain", "gz"])
def test_adversarial_fastq_files(env, gz):
    P = _pair(env, "fanc", "adv_%d" % gz)
    for name, text in _adversarial(AU.fanc_reads(3)).items():
        path = str(env["tmp"] / ("adv_%s.fastq%s" % (name, ".gz" if gz else "")))
        if gz:
            with gzip.open(path, "wb") as fh:
                fh.write(text.encode())
        else:
            with open(path, "wb") as fh:
                fh.write(text.encode())
        _check_fastq(P, path, tag=name, empty=not text)
        _check_sam(P, path, tag=name)


def test_sam_position_strand_and_chromosome(env):
    """refs with aln_chr / aln_start / aln_strand set (what a bowtie2-located amplicon carries): flag flip, reversed CIGAR
    elements, reverse-complemented sequence, reversed quality"""
    ref_names, refs, _ = env["caps"]["hdr"]
    refs2 = copy.deepcopy(refs)
    refs2[ref_names[0]].update(aln_chr="chr7", aln_start=1234, aln_strand="-")
    reads = AU.edited_reads(env["fanc"], refs[ref_names[0]]["include_idxs"])
    fq = AU.write_fastq(str(env["tmp"] / "strand.fastq"), reads)
    P = _pair(env, "hdr", "strand")
    _check_sam(P, fq, tag="strand", refs=refs2)
    _check_sam(P, fq, tag="strand_nodebug", refs=refs2, debug=False)


def test_sam_sort_failure_raises_like_the_reference(env, tmp_path):
    P = _pair(env, "fanc", "sortfail")
    old = os.environ["PATH"]
    bad = tmp_path / "badbin"
    bad.mkdir()
    (bad / "samtools").write_text("#!/bin/sh\nexit 3\n")
    os.chmod(str(bad / "samtools"), 0o755)
    os.environ["PATH"] = str(bad) + os.pathsep + old
    try:
        from crispresso2_b200 import annotate
        from CRISPResso2 import CRISPRessoShared
        with pytest.raises(CRISPRessoShared.BadParameterException, match="Bam sort failed. Command used: samtools sort"):
            annotate.process_single_fastq_write_bam_out(env["fq"], str(tmp_path / "x.bam"), "@HD\n", {}, P.ref_names,
                                                        copy.deepcopy(P.refs), P.args, [], str(tmp_path), process_fastq=P.pf)
    finally:
        os.environ["PATH"] = old


def test_materialised_entries_get_the_key_too(env):
    """an entry read before the write gets the key at once, after its other keys"""
    from crispresso2_b200 import annotate
    P = _pair(env, "fanc", "early")
    cache = {}
    seen = {}

    def pf(*a):
        out = P.pf(*a)
        k = next(iter(cache))
        seen["key"] = k
        cache[k]["aln_scores"]                                  # materialises this one entry
        return out

    annotate.process_fastq_write_out(env["fq"], str(env["tmp"] / "early.fastq.gz"), cache, P.ref_names, copy.deepcopy(P.refs), P.args,
                                     [], str(env["tmp"]), process_fastq=pf)
    v = cache[seen["key"]]
    assert dict.__contains__(v, "crispresso2_annotation") and list(dict.keys(v))[-1] == "crispresso2_annotation"


def test_score_text_matches_python_float_str(env):
    """str(k / 1000) for every score k in 0..100000 (round(100 m / n, 3) of the reference), as the device formats it"""
    import ctypes as C
    import numpy as np
    from crispresso2_b200 import _lib, annotate
    eng = env["engine"]
    n = 100001
    recs = np.zeros(n, dtype=_lib.REC_DTYPE)
    alns = np.zeros((n, 1), dtype=_lib.ALN_DTYPE)
    alns["score_milli"][:, 0] = np.arange(n)
    ops = np.zeros((n, 1, 1), dtype=np.uint64)
    meta = np.zeros((n, 1), dtype=np.uint32)
    edits = np.zeros((n, 1, 1), dtype=_lib.EDIT_DTYPE)
    off = np.zeros(n + 1, dtype=np.int64)
    bidx = np.arange(n, dtype=np.int32)
    amask = np.zeros(n, dtype=np.uint32)
    aname = np.full(n, -1, dtype=np.int16)
    label = np.full(n, -1, dtype=np.int32)
    rev = np.zeros(1, dtype=np.uint8)
    lens = np.asarray([4], dtype=np.int32)
    comp = annotate._comp256()
    h = C.c_void_p()
    rc = eng.L.c2b_annotate_build(eng.h, None, off.ctypes.data, n, bidx.ctypes.data, 1, 1, 1, recs.ctypes.data, alns.ctypes.data,
                                  ops.ctypes.data, meta.ctypes.data, edits.ctypes.data, amask.ctypes.data, aname.ctypes.data,
                                  label.ctypes.data, 1, annotate._cstrings(["R"]), rev.ctypes.data, 0, annotate._cstrings([]),
                                  annotate._cstrings(["ACGT"]), lens.ctypes.data, comp.ctypes.data, 0, 4096, C.byref(h))
    assert rc == 0
    try:
        o = np.ctypeslib.as_array(C.cast(eng.L.c2b_annotate_offsets(h), C.POINTER(C.c_int64)), shape=(n + 1,))
        text = C.string_at(eng.L.c2b_annotate_arena(h), int(o[-1])).decode()
        for k in range(n):
            s = str(k / 1000)
            assert text[o[k]:o[k + 1]] == " ALN=NA ALN_SCORES=%s ALN_DETAILS=R,,,%s" % (s, s), k
    finally:
        eng.L.c2b_annotate_free(h)


def test_cli_bam_output_is_byte_identical(tmp_path):
    """--bam_output through the launcher (cli_dropin_runner.py) against the unmodified CLI, with and without --debug"""
    import test_cli_dropin as T
    import build_emu
    lib = build_emu.build()
    path = AU.fake_samtools(str(tmp_path / "bin"))
    fanc, hdr = AU.amplicons()
    fq = AU.write_fastq(str(tmp_path / "FANC.fastq"), AU.fanc_reads())
    for extra in ([], ["--debug"]):
        argv = ["-r1", fq, "-a", fanc, "-g", G, "-e", hdr, "--bam_output"] + extra
        dirs = []
        for mode in ("reference", "b200"):
            # the SAM header carries the command line: both runs use the same relative output directory
            out = str(tmp_path / ("%s%d" % (mode, len(extra))))
            os.makedirs(out, exist_ok=True)
            p = subprocess.run([sys.executable, os.path.join(HERE, "cli_dropin_runner.py"), mode, lib if mode == "b200" else "default",
                                ".", "_vectors.json", "--"] + argv, capture_output=True, text=True, timeout=900, cwd=out,
                               env=dict(os.environ, PATH=path))
            assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
            dirs.append(out)
        a, b = T._snapshot(dirs[0]), T._snapshot(dirs[1])
        assert sorted(a) == sorted(b)
        assert [k for k in a if a[k] != b[k]] == []
        assert any(k.endswith("CRISPResso_output.bam") for k in a)
        assert any(k.endswith(".sam") for k in a) == bool(extra)
