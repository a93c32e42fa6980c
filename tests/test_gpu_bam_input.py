"""--bam_input on the sm_90a library: the GPU SAM front end (c2b_sam_dedup_gpu_buffer) against the host one byte for byte, the
function and CLI comparisons of tests/test_bam_input.py through the CUDA engine, and an annotation pass over several chunks."""
import copy
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import annotate_util as AU  # noqa: E402
import bam_util as BU  # noqa: E402
import test_bam_input as TB  # noqa: E402

pytestmark = pytest.mark.gpu


def same_dedup(a, b):
    assert a.n_reads == b.n_reads
    assert np.array_equal(a.off, b.off) and a.buf.tobytes() == b.buf.tobytes()
    assert np.array_equal(a.counts, b.counts) and np.array_equal(a.first_index, b.first_index)


def big_sam_text(n=1 << 20, seed=3):
    """~1 Mi SAM lines: bench-like reads with many duplicates, flags 0 / 16 / 4, bowtie2 tags, some CRLF endings"""
    rnd = np.random.default_rng(seed)
    base = ["".join(rnd.choice(list("ACGT"), size=int(rnd.integers(120, 260)))) for _ in range(4096)]
    pick = rnd.integers(0, len(base), size=n)
    pick[::7] = rnd.integers(0, 64, size=len(pick[::7]))        # a few reads carry most of the counts
    out = []
    for k in range(n):
        s = base[pick[k]]
        flag = (0, 16, 4)[k % 3]
        end = "\r\n" if k % 101 == 0 else "\n"
        out.append("M0:1:%d\t%d\tchr11\t%d\t42\t%dM\t*\t0\t0\t%s\t%s\tAS:i:-%d\tYT:Z:UU%s" % (k, flag, 1000 + k % 50, len(s), s,
                                                                                         "I" * len(s), k % 9, end))
    return "".join(out).encode()


def test_gpu_front_end_matches_the_host_one(monkeypatch):
    from crispresso2_b200 import fastq
    texts = dict(TB.adversarial_texts())
    texts["fixture"] = BU.sam_text_of(TB.FIXTURE, 0)
    texts["big"] = big_sam_text()
    for name, text in texts.items():
        same_dedup(fastq.dedup_sam(text, device=0), fastq.dedup_sam(text))
    TB.check_front_end(lambda t: fastq.dedup_sam(t, device=0), texts["fixture"])
    for name, text in TB.BAD_TEXTS.items():
        errs = []
        for dev in (0, None):
            try:
                fastq.dedup_sam(text, device=dev)
                errs.append(None)
            except (IndexError, fastq.FastqError) as ex:
                errs.append((type(ex), str(ex).split(": ", 1)[-1].split("(")[0]))
        assert errs[0] is not None and errs[0][0] == errs[1][0], (name, errs)
    monkeypatch.delenv("C2B_GPU_INGEST", raising=False)
    assert fastq._ingest_rule(len(texts["big"]), False, 0, None) == 0       # the CUDA build picks the device for this text


@pytest.fixture(scope="module")
def env(tmp_path_factory):
    from baseline import ref_shim
    from crispresso2_b200.engine import Engine
    if not AU.have_reference():
        pytest.skip("needs oracle/_ref/install")
    tmp = tmp_path_factory.mktemp("gpu_bam_input")
    old_path = os.environ["PATH"]
    os.environ["PATH"] = BU.fake_samtools(str(tmp / "bin"))
    try:
        fanc, hdr = AU.amplicons()
        fq = AU.write_fastq(str(tmp / "FANC.fastq"), AU.fanc_reads())
        caps = {"fanc": AU.capture(tmp, ["-r1", fq, "-a", fanc, "-g", TB.G]),
                "hdr": AU.capture(tmp, ["-r1", fq, "-a", fanc, "-g", TB.G, "-e", hdr])}
        import pe_case
        pe_fq = str(tmp / "pe_scaffold.fastq")
        ext, scaffold = pe_case.write_fastq(pe_fq, fanc)
        caps["pe"] = AU.capture(tmp, ["-r1", pe_fq, "-a", fanc, "--prime_editing_pegRNA_spacer_seq", TB.G,
                                      "--prime_editing_pegRNA_extension_seq", ext, "--prime_editing_pegRNA_scaffold_seq", scaffold])
        yield {"CORE": ref_shim.load_core(), "engine": Engine(0), "tmp": tmp, "caps": caps, "fanc": fanc, "pe_fq": pe_fq}
    finally:
        os.environ["PATH"] = old_path


@pytest.mark.parametrize("region,F", [("chr11:1024-1274", "4"), ("chr9:962-1198", "4"), ("", "0x10")], ids=["chr11", "chr9", "all"])
def test_gpu_fixture(env, region, F):
    TB.check_both(env, "fanc", TB.FIXTURE, region, "gfix_%s_%s" % (region.split(":")[0], F), samtools_exclude_flags=F)


def test_gpu_synthetic_hdr_and_scaffold(env):
    ref_names, refs, _ = env["caps"]["fanc"]
    reads = AU.edited_reads(env["fanc"], refs[ref_names[0]]["include_idxs"])
    p = TB.write_synthetic(str(env["tmp"] / "gedges.bam"), reads)
    TB.check_both(env, "fanc", p, "", "gedges", samtools_exclude_flags="4")
    TB.check_both(env, "hdr", p, "chr11", "ghdr", samtools_exclude_flags="4", expand_ambiguous_alignments=True)
    TB.check_both(env, "hdr", p, "chr11", "ghdr_first", assign_ambiguous_alignments_to_first_reference=True)
    lines = open(env["pe_fq"]).read().split("\n")
    pe = TB.write_synthetic(str(env["tmp"] / "gpe.bam"), [lines[k + 1] for k in range(0, len(lines) - 3, 4)])
    TB.check_both(env, "pe", pe, "", "gpe")


def test_gpu_bench_mix(env):
    """the bench's read mix (single amplicon) as a BAM with duplicates, through both functions"""
    import bench
    w = bench.Workload("single", 4096, 0)
    reads = [r.tobytes().decode() for r in w.buf.reshape(-1, 250)]
    reads = reads + reads[:1024]
    p = TB.write_synthetic(str(env["tmp"] / "gbench.bam"), reads)
    # the bench amplicon is not FANC: most reads do not align, which exercises not_aln at volume
    TB.check_both(env, "fanc", p, "", "gbench", samtools_exclude_flags="4")


def test_gpu_annotation_over_several_chunks(env):
    """the same annotations whether the device pass runs in one chunk or in chunks of 7 unique reads"""
    from crispresso2_b200 import annotate, bam
    ref_names, refs, args = env["caps"]["hdr"]
    reads = AU.edited_reads(env["fanc"], refs[ref_names[0]]["include_idxs"])
    p = TB.write_synthetic(str(env["tmp"] / "gchunks.bam"), reads)
    cache = {}
    bam.process_bam(p, "", str(env["tmp"] / "gchunks_out.bam"), cache, ref_names, copy.deepcopy(refs), args, [], str(env["tmp"]),
                    engine=env["engine"], aln_matrix=TB.matrix_of(env, args))
    one = annotate.Annotation(cache, refs, sam_optional=True)
    many = annotate.Annotation(cache, refs, sam_optional=True, chunk=7)
    assert one.n > 21
    assert one.arena.tobytes() == many.arena.tobytes() and np.array_equal(one.ann_off, many.ann_off)


def test_gpu_cli_bam_input_is_byte_identical(tmp_path):
    if not AU.have_reference():
        pytest.skip("needs oracle/_ref/install")
    TB.run_cli_pair(tmp_path, "default")
