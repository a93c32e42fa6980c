"""--base_editor_output allele tables at scale: the reference's get_upset_plot_counts and get_base_edit_dataframe_around_cut
(plots/data_prep.py, CRISPRessoShared.py of the package under oracle/_ref/install) against the drop-ins of
crispresso2_b200.base_edit, on the allele frame of a synthetic FASTQ (crispresso2_b200.synth via bench.Workload).

    python tools/base_edit_bench.py --reads 1048576 --config single|hdr [--reference-rows N] [--no-reference]

The frame is AlleleTable(...).to_dataframe() after the engine's process_fastq over the FASTQ, as main() sees it.  The targets
are the Cs of the first amplicon's guide (C -> T); the quilt runs on the rows of the first amplicon with conversion_nuc_from C,
as prep_base_edit_quilt calls it.  Prints one JSON line per config: the card's name and power limit, rows, the drop-ins' time
split into packing (numpy), device pass with its copies, host sum or grouping, and building the dict or frame; the reference's
time on the first --reference-rows rows (0: all) with the drop-ins' time on the same rows, and whether both results are equal
there.  Needs a GPU; writes only under a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def bench_frame(config, n, d, engine):
    """-> (df_alleles, bp_substitutions_arr, wt_ref_name, label) of `n` synthetic reads of bench.Workload(config)"""
    import bench
    from crispresso2_b200 import core, synth
    from crispresso2_b200.alleles import AlleleTable
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
    df = AlleleTable(cache).to_dataframe()
    wt = w.ref_names[0]
    ref = w.refs[wt]
    g = ref["cut_point"] + 3 - 20                               # the 20-nt guide ends 3 bp right of the cut (synth.amplicon_setup)
    bp = [(p, "C", "T") for p in range(g, g + 20) if ref["sequence"][p] == "C"]
    return df, bp, wt, w.label


def _timed(fn, *a, **kw):
    t = time.perf_counter()
    out = fn(*a, **kw)
    return out, time.perf_counter() - t


def run(config, n, with_reference, ref_rows, d):
    import logging
    import pandas as pd
    from crispresso2_b200 import base_edit, core, synth  # noqa: F401
    from vcf_bench import gpu_info
    logging.getLogger("CRISPResso2").setLevel(logging.ERROR)
    eng = core.get_engine(0)
    t0 = time.perf_counter()
    df, bp, wt, label = bench_frame(config, n, d, eng)
    sub = df.loc[df["Reference_Name"] == wt]
    res = {"config": config, "reads": n, "workload": label, "gpu": gpu_info(), "frame_build_s": time.perf_counter() - t0,
           "rows": len(df), "quilt_rows": len(sub), "targets": len(bp)}
    base_edit.get_upset_plot_counts(df, bp, wt, engine=eng)     # warm-up: engine, pinned and device buffers
    base_edit.get_base_edit_dataframe_around_cut(sub, "C", engine=eng)
    got_u, tu = _timed(base_edit.get_upset_plot_counts, df, bp, wt, engine=eng)
    tm = base_edit.get_upset_plot_counts.last_timings
    res["upset"] = {"total_s": tu, "pack_s": tm["pack"], "device_pass_and_copies_s": tm["device"], "host_sum_s": tm["host"],
                    "dict_s": tm["frame"], "precise_keys": len(got_u["precise_allele_counts"])}
    got_q, tq = _timed(base_edit.get_base_edit_dataframe_around_cut, sub, "C", engine=eng)
    tm = base_edit.get_base_edit_dataframe_around_cut.last_timings
    res["quilt"] = {"total_s": tq, "pack_s": tm["pack"], "device_pass_and_copies_s": tm["device"], "host_grouping_s": tm["host"],
                    "frame_s": tm["frame"], "groups": len(got_q)}
    if with_reference:
        import base_edit_util as U
        ref_upset, ref_quilt = U.reference()
        dfp = df.iloc[:ref_rows] if ref_rows else df
        subp = dfp.loc[dfp["Reference_Name"] == wt]
        res["reference_rows"] = len(dfp)
        for key, ref_fn, drop, a in (("upset", ref_upset, base_edit.get_upset_plot_counts, (dfp, bp, wt)),
                                     ("quilt", ref_quilt, base_edit.get_base_edit_dataframe_around_cut, (subp, "C"))):
            want, tr = _timed(ref_fn, *a)
            mine, td = _timed(drop, *a, engine=eng)
            if key == "upset":
                same = list(mine) == list(want) and all(
                    (list(mine[k].items()) == list(want[k].items())) if k.endswith("_allele_counts") else mine[k] == want[k] for k in want)
            else:
                try:
                    pd.testing.assert_frame_equal(mine, want, check_exact=True)
                    same = True
                except AssertionError:
                    same = False
            res[key].update({"reference_s": tr, "reference_us_per_row": 1e6 * tr / max(1, len(a[0])), "dropin_same_rows_s": td,
                             "speedup_same_rows": tr / td, "identical": same})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1 << 20)
    ap.add_argument("--config", default="single,hdr")
    ap.add_argument("--reference-rows", type=int, default=0, help="time the reference on this prefix of the frame (0: all)")
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        for config in a.config.split(","):
            print(json.dumps(run(config, a.reads, not a.no_reference, a.reference_rows, d)), flush=True)


if __name__ == "__main__":
    main()
