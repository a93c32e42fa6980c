"""--bam_input at scale: the reference's process_bam (single process) against crispresso2_b200.bam.process_bam on SAM text of the
bench read mix (bench.Workload), stage by stage.

    python tools/bam_bench.py [--records 1048576] [--ref-records 16384] [--config single,hdr] [--out DIR] [--lib PATH]

The records are rendered once to SAM text (flags 0 / 16, one contig); a `samtools` stand-in `cat`s that text (the header for
-H), so both functions read the same input at memory speed and the samtools decode is not part of either time.  The reference
aligns every unique read on the host, which is hours at 1 Mi records, so it runs on the first --ref-records records only, with
the drop-in on the same records; the outputs of that pair (.sam bytes, aln_stats, not_aln keys) are compared.  The drop-in alone
then runs on all --records records with its stages: pass-1 text (header + reading the samtools pipe), front end (SAM parse +
exact dedup), batch (core._process_uniques), annotation (device pass), pass-2 wait and writer.  The card's name and power limit
are read in the same run.  A real `samtools view` pass is timed only when one is on PATH; otherwise it is reported as not
measured.  Needs a GPU (or --lib with the emulator build, for a rehearsal at small sizes) and oracle/_ref/install; writes only
under a temporary directory (or --out for the JSON lines).
"""
import argparse
import copy
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


def render(w, n, path):
    """SAM text of the first n reads of the workload: flags 0 / 16 alternating, 250M on 'amplicon'"""
    buf = w.buf.reshape(-1, 250)[:n]
    qual = "I" * 250
    with open(path, "w") as fh:
        for k in range(n):
            fh.write("r%d\t%d\tamplicon\t1\t42\t250M\t*\t0\t0\t%s\t%s\tAS:i:0\tYT:Z:UU\n" % (k, 16 * (k & 1), buf[k].tobytes().decode(), qual))


def stand_in(bindir, header, text):
    os.makedirs(bindir, exist_ok=True)
    p = os.path.join(bindir, "samtools")
    with open(p, "w") as fh:
        fh.write('#!/bin/sh\nfor a in "$@"; do [ "$a" = -H ] && exec cat %s; done\nexec cat %s\n' % (header, text))
    os.chmod(p, 0o755)


def run(config, n, n_ref, lib, d):
    import logging
    import bench
    from baseline import ref_shim
    from crispresso2_b200 import bam, core
    from crispresso2_b200.engine import Engine
    from oracle import oracle as O
    CORE = ref_shim.load_core()
    for name in list(logging.root.manager.loggerDict) + ["CRISPResso2"]:
        if name.startswith("CRISPResso"):
            logging.getLogger(name).setLevel(logging.ERROR)
    w = bench.Workload(config, n, 0)
    args = types.SimpleNamespace(**vars(w.params))
    args.use_legacy_insertion_quantification = False
    args.prime_editing_pegRNA_scaffold_seq = args.prime_editing_pegRNA_extension_seq = ""
    args.needleman_wunsch_aln_matrix_loc = "EDNAFULL"
    args.n_processes = "1"
    args.samtools_exclude_flags = "4"
    refs = copy.deepcopy(w.refs)
    header = os.path.join(d, "header.sam")
    with open(header, "w") as fh:
        fh.write("@HD\tVN:1.0\tSO:unsorted\n@SQ\tSN:amplicon\tLN:250\n")
    eng = Engine(lib_path=lib) if lib else core.get_engine(0)
    matrix = O.make_matrix()
    res = {"config": config, "records": n, "workload": w.label, "gpu": gpu_info() if not lib else "emulator build (rehearsal)"}

    def drop_in(text, tag):
        stand_in(os.path.join(d, "bin"), header, text)
        cache = {}
        t0 = time.perf_counter()
        st, na = bam.process_bam("in.bam", "", os.path.join(d, tag + ".bam"), cache, w.ref_names, refs, args, [], d, engine=eng,
                                 aln_matrix=matrix)
        total = time.perf_counter() - t0
        stages = {k + ("_s" if not k.startswith("n_") else ""): v for k, v in bam.last_timings.items()}
        return total, stages, st, na

    # the pair on the first n_ref records
    small = os.path.join(d, "small.sam")
    render(w, n_ref, small)
    drop_in(small, "warm")                                      # warm-up: engine, allocations, page cache
    t_b, stages_b, st_b, na_b = drop_in(small, "b200_small")
    stand_in(os.path.join(d, "bin"), header, small)
    t0 = time.perf_counter()
    st_r, na_r = CORE.process_bam("in.bam", "", os.path.join(d, "ref_small.bam"), {}, w.ref_names, refs, args, [], d)
    t_r = time.perf_counter() - t0
    with open(os.path.join(d, "ref_small.bam.sam"), "rb") as fa, open(os.path.join(d, "b200_small.bam.sam"), "rb") as fb:
        identical = fa.read() == fb.read()
    res["pair"] = {"records": n_ref, "reference_s": t_r, "drop_in_s": t_b, "speedup": t_r / t_b, "drop_in_stages": stages_b,
                   "sam_identical": identical, "aln_stats_equal": st_r == st_b, "not_aln_keys_equal": list(na_r) == list(na_b)}
    # the drop-in alone at full size
    big = os.path.join(d, "big.sam")
    render(w, n, big)
    t_b, stages_b, _, _ = drop_in(big, "b200_big")
    res["drop_in_full"] = {"records": n, "total_s": t_b, "stages": stages_b, "records_per_s": n / t_b,
                           "sam_bytes": os.path.getsize(os.path.join(d, "b200_big.bam.sam"))}
    real = None
    for p in os.environ.get("C2B_REAL_PATH", "").split(os.pathsep):
        if p and os.path.exists(os.path.join(p, "samtools")):
            real = os.path.join(p, "samtools")
    res["samtools_view_pass"] = "not measured (no samtools on PATH)" if real is None else "see samtools_view_s"
    if real is not None:
        import bam_util as BU
        recs = [dict(qname="r%d" % k, flag=16 * (k & 1), rname="amplicon", pos=1, mapq=42, cigar="250M",
                     seq=w.buf.reshape(-1, 250)[k].tobytes().decode(), qual="I" * 250, tags=[]) for k in range(n)]
        bp = BU.write_bam(os.path.join(d, "big.bam"), "@HD\tVN:1.0\n", [("amplicon", 250)], recs)
        t0 = time.perf_counter()
        subprocess.run([real, "view", "-F", "4", bp], stdout=subprocess.DEVNULL, check=True)
        res["samtools_view_s"] = time.perf_counter() - t0
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1 << 20)
    ap.add_argument("--ref-records", type=int, default=16384)
    ap.add_argument("--config", default="single,hdr")
    ap.add_argument("--lib", default=None, help="engine library (default: the CUDA build on GPU 0)")
    ap.add_argument("--out", default=None, help="directory for the JSON lines (default: stdout only)")
    a = ap.parse_args()
    os.environ["C2B_REAL_PATH"] = os.environ.get("PATH", "")
    for config in a.config.split(","):
        d = tempfile.mkdtemp(prefix="c2b_bam_bench_")
        old = os.environ["PATH"]
        os.environ["PATH"] = os.path.join(d, "bin") + os.pathsep + old
        try:
            line = json.dumps(run(config, a.records, min(a.ref_records, a.records), a.lib, d))
        finally:
            os.environ["PATH"] = old
            shutil.rmtree(d, ignore_errors=True)
        print(line, flush=True)
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            with open(os.path.join(a.out, "bam_bench.jsonl"), "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
