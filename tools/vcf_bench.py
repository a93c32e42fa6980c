"""--vcf_output edit counts at scale: the reference's build_edit_counts (writers/vcf.py:172-212 of the package under
oracle/_ref/install) against the drop-in crispresso2_b200.vcf.build_edit_counts, on the allele frame of a synthetic FASTQ
(crispresso2_b200.synth via bench.Workload).

    python tools/vcf_bench.py --reads 1048576 --config single|hdr [--no-reference]

The frame holds one row per (unique read, aligned reference) with the columns main() builds for --vcf_output
(CRISPRessoCORE.py:3921-3945), from the engine's process_fastq over the FASTQ, without the AMBIGUOUS_ rows of the HDR workload
(the reference raises KeyError at the first of them that has edits).  Prints one JSON line per config: the card's
name and power limit, rows, edited rows, records and distinct keys, the reference's time, and the drop-in's time split into
packing (numpy), device pass with its copies (c2b_vcf_edit_counts up to the sum), the host sum, and building the dict.  Both
dicts are compared, keys in order.  Needs a GPU; writes only under a temporary directory.
"""
import argparse
import json
import os
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


def bench_frame(config, n, d, engine, amplicon_rows_only=True):
    """-> (df_alleles, amplicon_positions, label) of `n` synthetic reads of bench.Workload(config); amplicon_rows_only: without
    the AMBIGUOUS_ rows (the reference raises KeyError at the first one that has edits, as its CLI does)"""
    import bench
    import vcf_util as V
    from crispresso2_b200 import core, synth
    from oracle import oracle as O
    w = bench.Workload(config, n, 0)
    fq = os.path.join(d, "reads.fastq")
    synth.write_fastq_fast(fq, w.buf.reshape(n, -1))
    args = types.SimpleNamespace(**vars(w.params))
    args.use_legacy_insertion_quantification = False
    args.prime_editing_pegRNA_scaffold_seq = args.prime_editing_pegRNA_extension_seq = ""
    args.needleman_wunsch_aln_matrix_loc = "EDNAFULL"
    args.n_processes = "1"
    cache = {}
    core.process_fastq(fq, cache, w.ref_names, w.refs, args, [], d, engine=engine, aln_matrix=O.make_matrix())
    df = V.frame_from_cache(cache)
    amp = {nm: ("chr%d" % (1 + k % 2), 1000 + 100000 * k) for k, nm in enumerate(w.ref_names)}
    if amplicon_rows_only:
        df = df[df["Reference_Name"].isin(w.ref_names)].reset_index(drop=True)
    return df, amp, w.label


def run(config, n, with_reference, d):
    import logging
    import vcf_util as V
    from crispresso2_b200 import core, vcf
    logging.getLogger("CRISPResso2").setLevel(logging.ERROR)
    eng = core.get_engine(0)
    t0 = time.perf_counter()
    df, amp, label = bench_frame(config, n, d, eng)
    res = {"config": config, "reads": n, "workload": label, "gpu": gpu_info(), "frame_build_s": time.perf_counter() - t0,
           "rows": len(df), "edited_rows": int(len(vcf._edited_rows(df)))}
    vcf.build_edit_counts(df, amp, engine=eng)                  # warm-up: engine, pinned and device buffers
    t1 = time.perf_counter()
    got = vcf.build_edit_counts(df, amp, engine=eng)
    t2 = time.perf_counter()
    tm = vcf.build_edit_counts.last_timings
    res["dropin"] = {"total_s": t2 - t1, "pack_s": tm["pack"], "device_pass_and_copies_s": tm["device"], "sum_s": tm["sum"],
                     "dict_s": tm["dict"], "records": tm["records"], "distinct_keys": len(got)}
    if with_reference:
        ref = V.reference_vcf()
        t3 = time.perf_counter()
        want = ref.build_edit_counts(df, amp)
        t4 = time.perf_counter()
        res["reference_s"] = t4 - t3
        res["reference_us_per_edited_row"] = 1e6 * (t4 - t3) / max(1, res["edited_rows"])
        res["speedup"] = (t4 - t3) / (t2 - t1)
        res["identical"] = got == want and list(got) == list(want)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1 << 20)
    ap.add_argument("--config", default="single,hdr")
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        for config in a.config.split(","):
            print(json.dumps(run(config, a.reads, not a.no_reference, d)), flush=True)


if __name__ == "__main__":
    main()
