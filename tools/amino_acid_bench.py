"""--coding_seq amino-acid tables at scale: the reference's get_amino_acid_dataframe (CRISPRessoShared.py of the package under
oracle/_ref/install) against crispresso2_b200.amino_acids' drop-in, on the allele frame of a synthetic FASTQ
(crispresso2_b200.synth via bench.Workload).

    python tools/amino_acid_bench.py --reads 1048576 --config single|hdr [--reference-rows N] [--no-reference]

The frame is AlleleTable(...).to_dataframe() after the engine's process_fastq over the FASTQ, as main() sees it, restricted to
the first amplicon's rows (as prep_amino_acid_table passes it) without an N at or right of the exon start: the reference raises
KeyError on any such row.  The coding sequence starts 30 bp left of the cut and the amino-acid cut point is 10, with
BLOSUM62.  Prints one JSON line per config: the card's name and power limit, rows, distinct protein pairs, the drop-in's time
split into packing (numpy), row pass with its copies, pair dedup with the alignments, silent edits with the grouping, and the
frame; the reference's time on the first --reference-rows rows (0: all) with the drop-in's time on the same rows, and whether
both frames are equal there.  Needs a GPU; writes only under a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def bench_frame(config, n, d, engine):
    """-> (rows of the first amplicon, plot_left_idx, sequence_length, amino_acid_cut_point, label) of `n` synthetic reads"""
    import base_edit_bench
    df, _, wt, label = base_edit_bench.bench_frame(config, n, d, engine)
    import bench
    ref = bench.Workload(config, 8, 0).refs[wt]
    left = ref["cut_point"] - 30
    sub = df.loc[df["Reference_Name"] == wt]
    clean = [("N" not in a[rp.index(left):]) if left in rp else True
             for a, rp in zip(sub["Aligned_Sequence"].tolist(), sub["ref_positions"].tolist())]
    return sub.loc[clean], left, 40, 10, label


def _timed(fn, *a, **kw):
    t = time.perf_counter()
    out = fn(*a, **kw)
    return out, time.perf_counter() - t


def run(config, n, with_reference, ref_rows, d):
    import logging
    import pandas as pd
    from crispresso2_b200 import amino_acids, core
    from vcf_bench import gpu_info
    import amino_util as U
    logging.getLogger("CRISPResso2").setLevel(logging.ERROR)
    blosum = U.reference()[2]
    eng = core.get_engine(0)
    t0 = time.perf_counter()
    df, left, sl, cut, label = bench_frame(config, n, d, eng)
    res = {"config": config, "reads": n, "workload": label, "gpu": gpu_info(), "frame_build_s": time.perf_counter() - t0,
           "rows": len(df)}
    amino_acids.get_amino_acid_dataframe(df, left, sl, blosum, cut, engine=eng)       # warm-up: engine, pinned and device buffers
    got, tt = _timed(amino_acids.get_amino_acid_dataframe, df, left, sl, blosum, cut, engine=eng)
    tm = amino_acids.get_amino_acid_dataframe.last_timings
    res["dropin"] = {"total_s": tt, "pack_s": tm["pack"], "row_pass_and_copies_s": tm["rows"], "dedup_and_alignment_s": tm["align"],
                     "silent_edits_and_grouping_s": tm["group"], "frame_s": tm["frame"], "pairs": tm["pairs"], "groups": len(got)}
    if with_reference:
        dfp = df.iloc[:ref_rows] if ref_rows else df
        res["reference_rows"] = len(dfp)
        want, tr = _timed(U.reference()[0], dfp, left, sl, blosum, cut)
        mine, td = _timed(amino_acids.get_amino_acid_dataframe, dfp, left, sl, blosum, cut, engine=eng)
        try:
            pd.testing.assert_frame_equal(mine, want, check_exact=True)
            same = True
        except AssertionError:
            same = False
        res["dropin"].update({"reference_s": tr, "reference_us_per_row": 1e6 * tr / max(1, len(dfp)), "dropin_same_rows_s": td,
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
