"""--bam_input (crispresso2_b200.bam.process_bam) against the reference's own process_bam, on the CPU: the host SAM front end
against a Python restatement of the pass-1 loop, the function against the function (the .sam bytes, aln_stats, not_aln and
variantCache materialised in key order with the new keys, the count block against process_fastq's on the same reads), the
screening of reads outside the engine's contract, and the launcher against the unmodified CLI.  Emulator build; the function and
CLI comparisons need oracle/_ref/install.  SAM text comes from the samtools stand-in of bam_util (or a real samtools for the
CLI test when one is on PATH)."""
import copy
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))

import annotate_util as AU  # noqa: E402
import bam_util as BU  # noqa: E402

G = "GGAATCCCTTCTGCAGCACC"
FIXTURE = os.path.join(HERE, "golden", "Both.Cas9.fastq.smallGenome.bam")
need_ref = pytest.mark.skipif(not AU.have_reference(), reason="needs oracle/_ref/install (built by __graft_entry__.build())")
ROW = "q%d\t0\tchr11\t1\t0\t*\t*\t0\t0\t%s\tII\tAS:i:0"


def adversarial_texts():
    """SAM texts on the edges of the pass-1 loop's line rules -> bytes (None: expected to raise)"""
    r = lambda k, s: ROW % (k, s)
    return {
        "crlf": ("%s\r\n%s\r\n%s\r\n" % (r(0, "ACGT"), r(1, "ACGT"), r(2, "GG"))).encode(),
        "lone_cr": ("%s\r%s\r" % (r(0, "ACGT"), r(1, "AC"))).encode(),
        "mixed_ends": ("%s\r\n%s\n%s\r%s" % (r(0, "A"), r(1, "C"), r(2, "A"), r(3, "C"))).encode(),
        "trailing_space_tab": ("q\t0\tc\t1\t0\t*\t*\t0\t0\tACGT \t \nq\t0\tc\t1\t0\t*\t*\t0\t0\tACGT\t\t\n").encode(),
        "seq_last_field": ("q\t0\tc\t1\t0\t*\t*\t0\t0\tACGT  \r\nq\t0\tc\t1\t0\t*\t*\t0\t0\tACGT\x1f\nq\t0\tc\t1\t0\t*\t*\t0\t0\tAC GT\n").encode(),
        "star_and_duplicates": "".join(r(k, s) + "\n" for k, s in enumerate(["*", "ACGT", "*", "ACGT", "ACGT", "TT"])).encode(),
        "empty_seq": b"q\t0\tc\t1\t0\t*\t*\t0\t0\t\tII\n",
        "no_final_newline": ("%s\n%s" % (r(0, "ACGT"), r(1, "GGG"))).encode(),
        "empty": b"",
        "long_lines": "".join(r(k, "ACGT" * (30 + k)) + "\tXX:Z:" + "N" * 500 + "\n" for k in range(40)).encode(),
    }


BAD_TEXTS = {
    "short_line": ("%s\nq\t0\tc\t1\t0\t*\t*\t0\t0\n" % (ROW % (0, "AC"))).encode(),
    "nine_fields_and_blanks": b"q\t0\tc\t1\t0\t*\t*\t0\t\t  \n",
    "blank_line": ("%s\n\n%s\n" % (ROW % (0, "AC"), ROW % (1, "AC"))).encode(),
    "non_ascii": ("%s\n" % (ROW % (0, "ACé"))).encode(),
}


def check_front_end(dedup, text):
    """dedup(bytes) -> fastq.Dedup, against the Python loop"""
    want, n = BU.pass1_restated(text)
    dd = dedup(text)
    assert dd.n_reads == n
    assert dd.uniques == list(want)
    assert dd.counts.tolist() == list(want.values())


@pytest.fixture(scope="module")
def lib():
    import build_emu
    return build_emu.build()


def test_front_end_matches_the_python_loop(lib):
    from crispresso2_b200 import fastq
    for name, text in adversarial_texts().items():
        check_front_end(lambda t: fastq.dedup_sam(t, lib_path=lib), text)
    for F, region in ((4, "chr11:1024-1274"), (0, None), (0x10, "chr9:962-1198")):
        check_front_end(lambda t: fastq.dedup_sam(t, lib_path=lib, n_threads=3), BU.sam_text_of(FIXTURE, F, region))


def test_front_end_errors(lib):
    from crispresso2_b200 import fastq
    for name in ("short_line", "nine_fields_and_blanks", "blank_line"):
        with pytest.raises(IndexError):
            BU.pass1_restated(BAD_TEXTS[name])
        with pytest.raises(IndexError, match="fewer than 10"):
            fastq.dedup_sam(BAD_TEXTS[name], lib_path=lib)
    with pytest.raises(fastq.FastqError, match="non-ASCII"):
        fastq.dedup_sam(BAD_TEXTS["non_ascii"], lib_path=lib)


def test_front_end_choice_follows_the_fastq_rule(lib, monkeypatch):
    """the emulator build has no device front end: process_bam's choice falls to the host threads, as process_fastq's does"""
    from crispresso2_b200 import fastq
    monkeypatch.delenv("C2B_GPU_INGEST", raising=False)
    text = BU.sam_text_of(FIXTURE, 4)
    check_front_end(lambda t: fastq.dedup_for_process_bam(t, 0, lib), text)
    monkeypatch.setenv("C2B_GPU_INGEST", "1")
    with pytest.raises(fastq.FastqError, match="not built"):
        fastq.dedup_for_process_bam(text, 0, lib)


def test_bam_util_round_trip(tmp_path):
    """the BAM writer and reader of the stand-in agree with each other"""
    recs = [dict(qname="a", flag=0, rname="chr1", pos=5, mapq=42, cigar="3M1I2M2D1M", seq="ACGTACG", qual="IIIIIII",
                 tags=[("AS", "i", -5), ("NM", "i", 3), ("YT", "Z", "UU"), ("XF", "f", 1.5), ("XA", "A", "x")]),
            dict(qname="b", flag=4, rname="*", pos=0, mapq=0, cigar="*", seq="NNAC", qual="*", tags=[])]
    p = BU.write_bam(str(tmp_path / "x.bam"), "@HD\tVN:1.0\n", [("chr1", 100)], recs)
    header, refs, got = BU.read_bam(p)
    assert header == "@HD\tVN:1.0\n" and refs == [("chr1", 100)]
    assert got[0][0] == "a\t0\tchr1\t5\t42\t3M1I2M2D1M\t*\t0\t0\tACGTACG\tIIIIIII\tAS:i:-5\tNM:i:3\tYT:Z:UU\tXF:f:1.5\tXA:A:x\n"
    assert got[1][0] == "b\t4\t*\t0\t0\t*\t*\t0\t0\tNNAC\t*\n"
    assert got[0][3:] == (4, 12)
    assert BU.sam_text_of(p, 0, "chr1:12-20") == got[0][0].encode() and BU.sam_text_of(p, 0, "chr1:13") == b""
    assert BU.sam_text_of(p, 4) == got[0][0].encode() and BU.parse_flags("0x10") == 16 and BU.parse_flags("020") == 16


# ------------------------------------------------------------------------------------------------ function against function
def synthetic_records(reads, seed=5):
    """records cycling through flags 0 / 16 / 4 on chr11, bowtie2-like tags; every third read also appears once as an unmapped
    (flag 4) record, and a few flag-4 records carry reads no included record has"""
    rnd = np.random.default_rng(seed)
    recs = []
    for k, s in enumerate(reads):
        flag = (0, 16, 4, 0, 16)[k % 5]
        mapped = not flag & 4
        recs.append(dict(qname="r%d" % k, flag=flag, rname="chr11" if mapped else "*", pos=1030 + k % 7 if mapped else 0,
                         mapq=42 if mapped else 0, cigar="%dM" % len(s) if mapped else "*", seq=s, qual="I" * len(s),
                         tags=[("AS", "i", -(k % 9)), ("XN", "i", 0), ("YT", "Z", "UU")] if mapped else [("YT", "Z", "UU")]))
        if k % 3 == 0:
            recs.append(dict(qname="u%d" % k, flag=4, rname="*", pos=0, mapq=0, cigar="*", seq=s, qual="F" * len(s), tags=[]))
    for k in range(4):
        s = "".join(rnd.choice(list("ACGT"), size=90))
        recs.append(dict(qname="x%d" % k, flag=4, rname="*", pos=0, mapq=0, cigar="*", seq=s, qual="F" * len(s), tags=[]))
    return recs


def write_synthetic(path, reads):
    return BU.write_bam(path, "@HD\tVN:1.0\tSO:unsorted\n@SQ\tSN:chr11\tLN:5000\n", [("chr11", 5000)], synthetic_records(reads))


@pytest.fixture(scope="module")
def env(tmp_path_factory, lib):
    from baseline import ref_shim
    from crispresso2_b200.engine import Engine
    tmp = tmp_path_factory.mktemp("bam_input")
    old_path = os.environ["PATH"]
    os.environ["PATH"] = BU.fake_samtools(str(tmp / "bin"))
    try:
        fanc, hdr = AU.amplicons()
        fq = AU.write_fastq(str(tmp / "FANC.fastq"), AU.fanc_reads())
        caps = {"fanc": AU.capture(tmp, ["-r1", fq, "-a", fanc, "-g", G]),
                "hdr": AU.capture(tmp, ["-r1", fq, "-a", fanc, "-g", G, "-e", hdr])}
        import pe_case
        pe_fq = str(tmp / "pe_scaffold.fastq")
        ext, scaffold = pe_case.write_fastq(pe_fq, fanc)
        caps["pe"] = AU.capture(tmp, ["-r1", pe_fq, "-a", fanc, "--prime_editing_pegRNA_spacer_seq", G,
                                      "--prime_editing_pegRNA_extension_seq", ext, "--prime_editing_pegRNA_scaffold_seq", scaffold])
        yield {"CORE": ref_shim.load_core(), "engine": Engine(lib_path=lib), "tmp": tmp, "caps": caps, "fanc": fanc,
               "pe_fq": pe_fq}
    finally:
        os.environ["PATH"] = old_path


def matrix_of(env, args):
    from crispresso2_b200 import core
    loc = args.needleman_wunsch_aln_matrix_loc
    return core.read_matrix(loc if os.path.isabs(loc) else os.path.join(env["CORE"]._ROOT, loc))


def run_both(env, which, bam_path, region, tag, **flags):
    """the reference's process_bam and bam.process_bam on the same input -> (ref result, ours, caches, .sam bytes)"""
    from crispresso2_b200 import bam, core
    ref_names, refs, args = env["caps"][which]
    args = copy.copy(args)
    for k, v in flags.items():
        setattr(args, k, v)
    d = env["tmp"] / tag
    d.mkdir(exist_ok=True)
    matrix = matrix_of(env, args)
    old_argv = sys.argv
    sys.argv = ["CRISPResso", "--bam_input", "x.bam"]             # @PG CL: the same command line for both
    try:
        cache_r, cache_b = {}, {}
        res_r = env["CORE"].process_bam(bam_path, region, str(d / "ref.bam"), cache_r, ref_names, copy.deepcopy(refs), args, [], str(d))
        res_b = bam.process_bam(bam_path, region, str(d / "b200.bam"), cache_b, ref_names, copy.deepcopy(refs), args, [], str(d),
                                engine=env["engine"], aln_matrix=matrix)
    finally:
        sys.argv = old_argv
    sams = [open(str(d / p), "rb").read() for p in ("ref.bam.sam", "b200.bam.sam")]
    assert not os.path.exists(str(d / "b200.bam"))
    return res_r, res_b, cache_r, cache_b, sams, (ref_names, refs, args, matrix, d)


def check_both(env, which, bam_path, region, tag, **flags):
    from crispresso2_b200 import core, lazy
    res_r, res_b, cache_r, cache_b, sams, (ref_names, refs, args, matrix, d) = run_both(env, which, bam_path, region, tag, **flags)
    assert sams[0] == sams[1]
    assert res_r[0] == res_b[0]
    lazies = [v for v in list(cache_b.values()) + list(res_b[1].values()) if isinstance(v, lazy.LazyVariant)]
    assert all(getattr(v, "_k", -1) >= 0 for v in lazies)        # nothing materialised by the call
    for a, b, key in ((cache_r, cache_b, "crispresso2_annotation"), (res_r[1], res_b[1], "crispresso_sam_optional_fields")):
        assert list(a.keys()) == list(b.keys())
        for s in a:
            AU.same(a[s], b[s], "%s[%s..]" % (key, s[:12]))
            assert list(b[s].keys())[-1] == key
    # the count block: the one process_fastq accumulates for the same pass-1 reads
    text = BU.sam_text_of(bam_path, BU.parse_flags(args.samtools_exclude_flags), region or None)
    reads = [line.split("\t")[9] for line in text.decode().split("\n") if line]
    fq = AU.write_fastq(str(d / "pass1.fastq"), reads)
    cache_f = {}
    core.process_fastq(fq, cache_f, ref_names, copy.deepcopy(refs), args, [], str(d), engine=env["engine"], aln_matrix=matrix)
    bb, bf = core.quantify(cache_b), core.quantify(cache_f)
    assert bb.class_counts() == bf.class_counts()
    want_classes = {}
    for v in cache_r.values():
        want_classes[v["class_name"]] = want_classes.get(v["class_name"], 0) + v["count"]
    if not args.expand_ambiguous_alignments:
        assert bb.class_counts() == want_classes
    for r in bb.ref_names:
        Vb, Vf = bb.vectors(r), bf.vectors(r)
        assert sorted(Vb) == sorted(Vf) and all(np.array_equal(Vb[k], Vf[k]) for k in Vb), r
        assert bb.scalars(r) == bf.scalars(r), r
    return res_r, res_b, cache_r, sams[0]


@need_ref
@pytest.mark.parametrize("region,F", [("chr11:1024-1274", "4"), ("chr9:962-1198", "4"), ("", "4"), ("chr11:1024-1274", "0"),
                                      ("", "0x10")], ids=["chr11", "chr9", "no_region", "F0", "F0x10"])
def test_fixture(env, region, F):
    res_r, _, cache_r, sam = check_both(env, "fanc", FIXTURE, region, "fix_%s_%s" % (region.split(":")[0], F),
                                        samtools_exclude_flags=F)
    assert sam.count(b"\n") > 3
    if region == "chr9:962-1198":                               # HEK3 reads against the FANC amplicon: not aligned
        assert len(res_r[1]) > 0


@need_ref
def test_synthetic_mix_excluded_records_and_global_subs_quirk(env):
    ref_names, refs, _ = env["caps"]["fanc"]
    reads = AU.edited_reads(env["fanc"], refs[ref_names[0]]["include_idxs"])
    p = write_synthetic(str(env["tmp"] / "edges.bam"), reads)
    res_r, res_b, cache_r, sam = check_both(env, "fanc", p, "", "edges", samtools_exclude_flags="4")
    # records excluded by -F that share a read with an included one are written in pass 2; the others are dropped
    assert b"\nu0\t4\t" in sam and b"\nx0\t" not in sam
    # the N_GLOBAL_SUBS quirk shows: an aligned read with substitutions seen more than once
    assert any(v["count"] > 1 and v["variant_" + v["best_match_name"]]["substitution_n"] > 0 for v in cache_r.values())


@need_ref
@pytest.mark.parametrize("flags", [{}, {"expand_ambiguous_alignments": True}, {"assign_ambiguous_alignments_to_first_reference": True}],
                         ids=["default", "expand", "assign_first"])
def test_hdr(env, flags):
    ref_names, refs, _ = env["caps"]["hdr"]
    reads = AU.edited_reads(env["fanc"], refs[ref_names[0]]["include_idxs"], seed=3)
    p = write_synthetic(str(env["tmp"] / "hdr.bam"), reads)
    check_both(env, "hdr", p, "chr11", "hdr_" + "_".join(flags), samtools_exclude_flags="4", **flags)


@need_ref
def test_prime_editing_scaffold(env):
    lines = open(env["pe_fq"]).read().split("\n")
    reads = [lines[k + 1] for k in range(0, len(lines) - 3, 4)]
    p = write_synthetic(str(env["tmp"] / "pe.bam"), reads)
    _, _, cache_r, _ = check_both(env, "pe", p, "", "pe")
    assert any(v["class_name"] == "Scaffold-incorporated" for v in cache_r.values())


@need_ref
def test_screening_reads_outside_the_contract(env, caplog):
    """SEQ '*' and lower-case reads: a warning, not_aln entries with the short annotation; "error" raises before any launch"""
    from crispresso2_b200 import bam, core
    ref_names, refs, args = env["caps"]["fanc"]
    good = AU.fanc_reads(30)
    text = "".join(ROW % (k, s) + "\n" for k, s in enumerate(good + ["*", good[0].lower(), "*"])).encode()
    sam_in = str(env["tmp"] / "screen.sam")
    with open(sam_in, "wb") as fh:
        fh.write(b"@HD\tVN:1.0\n" + text)
    out = str(env["tmp"] / "screen.bam")
    cache = {}
    with caplog.at_level("WARNING", logger="CRISPResso2"):
        st, not_aln = bam.process_bam(sam_in, "", out, cache, ref_names, copy.deepcopy(refs), args, [], str(env["tmp"]),
                                      engine=env["engine"], aln_matrix=matrix_of(env, args))
    assert "outside the engine's contract" in caplog.text
    for s, c in (("*", 2), (good[0].lower(), 1)):
        assert not_aln[s]["count"] == c and not_aln[s]["crispresso_sam_optional_fields"] == bam.SAM_NA
        assert s not in cache
    lines = open(out + ".sam", "rb").read().decode().split("\n")
    assert sum(line.endswith("\t" + bam.SAM_NA) for line in lines) == 3
    n_launch = env["engine"].launch_count()
    with pytest.raises(core.EngineError, match="outside the engine's contract"):
        bam.process_bam(sam_in, "", out, {}, ref_names, copy.deepcopy(refs), args, [], str(env["tmp"]), engine=env["engine"],
                        aln_matrix=matrix_of(env, args), on_out_of_contract="error")
    assert env["engine"].launch_count() == n_launch


@need_ref
def test_empty_selection_raises_like_the_reference(env):
    from crispresso2_b200 import bam
    ref_names, refs, args = env["caps"]["fanc"]
    with pytest.raises(UnboundLocalError):
        env["CORE"].process_bam(FIXTURE, "chr11:1-5", str(env["tmp"] / "e_ref.bam"), {}, ref_names, copy.deepcopy(refs), args, [],
                                str(env["tmp"]))
    with pytest.raises(UnboundLocalError):
        bam.process_bam(FIXTURE, "chr11:1-5", str(env["tmp"] / "e_b200.bam"), {}, ref_names, copy.deepcopy(refs), args, [],
                        str(env["tmp"]), engine=env["engine"], aln_matrix=matrix_of(env, args))


# ------------------------------------------------------------------------------------------------ CLI
def cli_paths(tmp_path):
    paths = [("stand-in", BU.fake_samtools(str(tmp_path / "bin")))]
    if shutil.which("samtools"):
        paths.append(("samtools", os.environ["PATH"]))
    return paths


def run_cli_pair(tmp_path, lib, extra=()):
    import test_cli_dropin as T
    fanc, _ = AU.amplicons()
    for label, path in cli_paths(tmp_path):
        for keep in ([], ["--keep_intermediate"]):
            argv = ["--bam_input", FIXTURE, "--bam_chr_loc", "chr11:1024-1274", "-a", fanc, "-g", G] + keep + list(extra)
            dirs = []
            for mode in ("reference", "b200"):
                out = str(tmp_path / ("%s_%s_%d" % (label, mode, len(keep))))
                os.makedirs(out, exist_ok=True)
                p = subprocess.run([sys.executable, os.path.join(HERE, "bam_cli_runner.py"), mode, lib if mode == "b200" else "default",
                                    ".", "--"] + argv, capture_output=True, text=True, timeout=900, cwd=out, env=dict(os.environ, PATH=path))
                assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
                dirs.append(out)
            a, b = T._snapshot(dirs[0]), T._snapshot(dirs[1])
            assert sorted(a) == sorted(b)
            assert [k for k in a if a[k] != b[k]] == []
            assert any(k.endswith(".sam") for k in a) == bool(keep)


@need_ref
def test_cli_bam_input_is_byte_identical(tmp_path, lib):
    """--bam_input through the launcher against the unmodified CLI, with and without --keep_intermediate"""
    run_cli_pair(tmp_path, lib)
