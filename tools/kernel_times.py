"""Per-kernel device time of the flagship step (bench.py's `single` config through c2b_align_batch_device).

Runs the workload under torch.profiler (CUDA activity only, nothing else timed in this process) and prints the mean
time per launch of every kernel by name, the launch order of one step, the diagonal tier's read counts per step and
the card with its power limit: means over the profiled steps.

  python tools/kernel_times.py [--reads 1048576] [--steps 20] [--warmup 3] [--mix bench|proved|unproved] [--json OUT]

--mix replaces the bench's reads (same amplicon, same count): `proved` = reads as long as the amplicon with 0-2
substitutions and no gap (what the diagonal tier proves), `unproved` = the bench's deletion and insertion templates only.
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info(index):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, smax = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_w": float(plim), "max_sm_clock_mhz": float(smax)}
    except Exception as exc:                     # nvidia-smi missing or unparsable: the numbers still print
        return {"name": None, "error": str(exc)}


def mix_reads(mix, ref, n):
    """[n, 250] uint8 reads of --mix `proved` / `unproved` against the bench amplicon (fixed seed)"""
    import numpy as np
    from crispresso2_b200 import synth
    rng = np.random.default_rng(2024)
    amp = ref["sequence"]
    if mix == "unproved":                        # the bench's deletion (25 %) and insertion (10 %) templates, nothing else
        return synth.synth_reads_fast(rng, amp, n, 250, del_frac=0.25 / 0.35, ins_frac=0.10 / 0.35, cut=ref["cut_point"])
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    out = np.tile(np.frombuffer(amp.encode(), dtype=np.uint8), (n, 1))
    for k in range(2):                           # 0, 1 or 2 substitutions per read, each to a different base
        rows = np.nonzero(rng.integers(0, 3, size=n) > k)[0]
        cols = rng.integers(0, out.shape[1], size=len(rows))
        old = out[rows, cols]
        new = acgt[rng.integers(0, 4, size=len(rows))]
        new = np.where(new == old, acgt[(np.searchsorted(acgt, new) + 1) % 4], new)
        out[rows, cols] = new
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mix", default="bench", choices=["bench", "proved", "unproved"])
    ap.add_argument("--json", help="also write the table as JSON here")
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench import Workload
    from crispresso2_b200.engine import Engine
    from oracle import oracle as O

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    n = args.reads
    w = Workload("single", n, 0)
    eng = Engine(0)
    P = w.params
    if args.mix != "bench":
        w.buf = mix_reads(args.mix, w.refs["Reference"], n).reshape(-1)
    eng.configure(w.refs, w.ref_names, O.make_matrix(), P.needleman_wunsch_gap_open, P.needleman_wunsch_gap_extend,
                  P.aln_seed_count, P.aln_seed_min, w.flags, "ACGTN", 12)
    W = eng.string_width(w.max_len)
    L = eng.L
    d_reads = torch.from_numpy(np.ascontiguousarray(w.buf)).to(dev)
    d_off = torch.from_numpy(w.off).to(dev)
    d_recs = torch.empty(n * 16, dtype=torch.uint8, device=dev)
    d_alns = torch.empty(n * 32, dtype=torch.uint8, device=dev)
    d_str = torch.empty(n * 2 * W, dtype=torch.uint8, device=dev)
    d_ed = torch.empty(n * 12 * 8, dtype=torch.uint8, device=dev)

    def step():
        rc = L.c2b_align_batch_device(eng.h, d_reads.data_ptr(), d_off.data_ptr(), n, w.max_len, None, None, None,
                                      d_recs.data_ptr(), d_alns.data_ptr(), d_str.data_ptr(), d_ed.data_ptr())
        if rc != 0:
            raise RuntimeError(L.c2b_last_error(eng.h).decode())

    for _ in range(args.warmup):
        eng.counts_reset()
        step()
    eng.sync()
    torch.cuda.synchronize(dev)
    eng.counts_reset()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        eng.sync()
        torch.cuda.synchronize(dev)

    # kernels in launch order; every step launches the same sequence, so position k of a step names one launch (the ALIGN
    # kernel runs twice per step: narrow tier, then wide ring)
    evs = [ev for ev in prof.events() if ev.device_type.name == "CUDA" and "c2b_" in ev.name]
    evs.sort(key=lambda ev: ev.time_range.start)
    if not evs or len(evs) % args.steps:
        raise SystemExit("kernel_times: %d kernel records for %d steps" % (len(evs), args.steps))
    per_step = len(evs) // args.steps
    per = defaultdict(list)
    names = []
    for k, ev in enumerate(evs):
        short = ev.name.split("(")[0].replace("void ", "")
        key = (k % per_step, short)
        if k < per_step:
            names.append(key)
        per[key].append(ev.time_range.elapsed_us() / 1000.0)
    rows = []
    total = 0.0
    for key in names:
        v = per[key]
        if len(v) != args.steps:
            raise SystemExit("kernel_times: launch sequence differs between steps")
        ms = sum(v) / len(v)
        total += ms
        rows.append({"launch": key[0] + 1, "kernel": key[1], "ms_per_launch": ms})

    diag = None
    if hasattr(L, "c2b_diag_counts"):
        import ctypes as C
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        if L.c2b_diag_counts(eng.h, C.byref(a), C.byref(b), C.byref(c)) == 0:
            diag = {"proved": a.value // args.steps, "tier1": b.value // args.steps, "tier2": c.value // args.steps}
    info = card_info(0)
    print("card: %s, power limit %s W, max SM clock %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("max_sm_clock_mhz")))
    print("%d reads x 250 bp (mix %s), %d profiled steps after %d warm-up steps; C2B_NO_DIAG=%s" % (
        n, args.mix, args.steps, args.warmup, os.environ.get("C2B_NO_DIAG", "")))
    print("| # | kernel | ms / launch | share |")
    print("|---|---|---|---|")
    for r in rows:
        print("| %d | %s | %.3f | %.0f %% |" % (r["launch"], r["kernel"], r["ms_per_launch"], 100.0 * r["ms_per_launch"] / total if total else 0.0))
    print("| | sum of kernel times per step | %.3f | |" % total)
    if diag is not None:
        print("reads per step: %d proved on the diagonal (%.1f %%), %d to the narrow tier, %d to the wide ring" %
              (diag["proved"], 100.0 * diag["proved"] / n, diag["tier1"], diag["tier2"]))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": info, "reads": n, "steps": args.steps, "mix": args.mix, "no_diag": os.environ.get("C2B_NO_DIAG", ""),
                       "kernels": rows, "total_ms_per_step": total, "diag_counts": diag}, fh, indent=1)


if __name__ == "__main__":
    main()
