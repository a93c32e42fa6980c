"""--fastq_output / --bam_output at scale: the reference's wrappers over the engine's lazy cache (what the launcher ran before
crispresso2_b200.annotate) against the native path, on a synthetic FASTQ (crispresso2_b200.synth via bench.Workload).

    python tools/annotate_bench.py --reads 1048576 --config single|hdr [--no-reference] [--out DIR]

Prints one JSON line per config.  Stages of the native path: process_fastq (shared by both paths, timed once per path), the
device annotation pass (c2b_annotate_build: chunk copies, size / scan / write kernels, copies back), and the writer
(c2b_annotate_write_fastq: re-read + record assembly + gzip deflate + file write, fused per host thread; the FASTQ writer's
deflate alone is also timed on the same text).  Both outputs are compared (decompressed FASTQ, SAM text).  `samtools` is a
copying stand-in here (sort / index are the same external command on both paths and are not timed).  Needs a GPU and
oracle/_ref/install; writes only under a temporary directory (or --out).
"""
import argparse
import copy
import ctypes as C
import functools
import gzip
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=60).stdout.strip()
    except OSError:
        return "unknown"


def run(config, n, with_reference, d):
    import logging
    import numpy as np
    import bench
    import annotate_util as AU
    from baseline import ref_shim
    from crispresso2_b200 import annotate, core, synth
    from oracle import oracle as O
    logging.getLogger("CRISPResso2").setLevel(logging.ERROR)
    CORE = ref_shim.load_core()
    for name in list(logging.root.manager.loggerDict):
        if name.startswith("CRISPResso"):
            logging.getLogger(name).setLevel(logging.ERROR)
    w = bench.Workload(config, n, 0)
    fq = os.path.join(d, "reads.fastq")
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
    header = AU.bam_header(w.ref_names, refs)
    eng = core.get_engine(0)
    pf0 = functools.partial(core.process_fastq, engine=eng, aln_matrix=O.make_matrix())
    t_pf = {}

    def pf(*a):
        t0 = time.perf_counter()
        out = pf0(*a)
        t_pf["s"] = time.perf_counter() - t0
        return out

    pf(fq, {}, w.ref_names, refs, args, [], d)                 # warm-up: page cache, engine, allocations
    res = {"config": config, "reads": n, "workload": w.label, "gpu": gpu_info()}
    # native path, stage by stage (the calls of annotate.process_fastq_write_out / process_single_fastq_write_bam_out)
    cache = {}
    t0 = time.perf_counter()
    pf(fq, cache, w.ref_names, refs, args, [], d)
    t1 = time.perf_counter()
    A = annotate.Annotation(cache, refs)
    t2 = time.perf_counter()
    out_b = os.path.join(d, "b200.fastq.gz")
    A.write_fastq(fq, out_b)
    t3 = time.perf_counter()
    A.attach(cache, "crispresso2_annotation", A.annotation_of)
    t4 = time.perf_counter()
    text = bytes(A.arena[:min(len(A.arena), 64 << 20)])        # deflate alone, same level, one thread, on 64 MB of annotation text
    t5 = time.perf_counter()
    z = gzip.compress(text, compresslevel=6)
    t6 = time.perf_counter()
    res["native_fastq"] = {"process_fastq_s": t1 - t0, "annotate_device_pass_s": t2 - t1, "write_s": t3 - t2, "attach_s": t4 - t3,
                           "total_s": t4 - t0, "output_bytes": os.path.getsize(out_b), "annotation_bytes": int(A.ann_off[-1]),
                           "deflate_1thread_MB_per_s": len(text) / (t6 - t5) / 1e6 if t6 > t5 else None,
                           "unique_reads": int(A.n)}
    del z
    cache = {}
    A = None
    bam_b = os.path.join(d, "b200.bam")
    t0 = time.perf_counter()
    annotate.process_single_fastq_write_bam_out(fq, bam_b, header, cache, w.ref_names, refs, args, [], d, process_fastq=pf)
    res["native_sam"] = {"total_s": time.perf_counter() - t0, "process_fastq_s": t_pf["s"], "sam_bytes": os.path.getsize(bam_b + ".sam")}
    cache = None
    if with_reference:
        saved = CORE.process_fastq
        CORE.process_fastq = pf
        try:
            out_r = os.path.join(d, "ref.fastq.gz")
            t0 = time.perf_counter()
            CORE.process_fastq_write_out(fq, out_r, {}, w.ref_names, refs, args, [], d)
            dt = time.perf_counter() - t0
            res["reference_fastq"] = {"total_s": dt, "process_fastq_s": t_pf["s"], "write_loop_s": dt - t_pf["s"]}
            with gzip.open(out_r, "rb") as fa, gzip.open(out_b, "rb") as fb:
                res["fastq_identical"] = fa.read() == fb.read()
            os.remove(out_r)
            bam_r = os.path.join(d, "ref.bam")
            t0 = time.perf_counter()
            CORE.process_single_fastq_write_bam_out(fq, bam_r, header, {}, w.ref_names, refs, args, [], d)
            dt = time.perf_counter() - t0
            res["reference_sam"] = {"total_s": dt, "process_fastq_s": t_pf["s"], "write_loop_s": dt - t_pf["s"]}
            with open(bam_r + ".sam", "rb") as fa, open(bam_b + ".sam", "rb") as fb:
                res["sam_identical"] = fa.read() == fb.read()
        finally:
            CORE.process_fastq = saved
        nf, nsam = res["native_fastq"], res["native_sam"]
        res["speedup_fastq_after_process_fastq"] = res["reference_fastq"]["write_loop_s"] / (nf["total_s"] - nf["process_fastq_s"])
        res["speedup_sam_after_process_fastq"] = res["reference_sam"]["write_loop_s"] / (nsam["total_s"] - nsam["process_fastq_s"])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1 << 20)
    ap.add_argument("--config", default="single,hdr")
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the JSON lines (default: stdout only)")
    a = ap.parse_args()
    import annotate_util as AU
    for config in a.config.split(","):
        d = tempfile.mkdtemp(prefix="c2b_annotate_bench_")
        old = os.environ["PATH"]
        os.environ["PATH"] = AU.fake_samtools(os.path.join(d, "bin"))
        try:
            line = json.dumps(run(config, a.reads, not a.no_reference, d))
        finally:
            os.environ["PATH"] = old
            shutil.rmtree(d, ignore_errors=True)
        print(line, flush=True)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "annotate_bench.jsonl"), "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
