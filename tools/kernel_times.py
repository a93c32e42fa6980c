"""Per-kernel device time of the flagship step (bench.py's `single` config through c2b_align_batch_device).

Runs the workload under torch.profiler (CUDA activity only, nothing else timed in this process) and prints the mean
time per launch of every kernel by name, the launch order of one step, the diagonal tier's read counts per step and
the card with its power limit: means over the profiled steps.

  python tools/kernel_times.py [--reads 1048576] [--steps 20] [--warmup 3] [--mix bench|proved|unproved] [--route-report] [--json OUT]
  python tools/kernel_times.py --one-kernel coding1,coding3,amp8,nosplit [--reads 1048576] [--steps 20] [--warmup 3] [--json OUT]

--mix replaces the bench's reads (same amplicon, same count): `proved` = reads as long as the amplicon with 0-2
substitutions and no gap (what the diagonal tier proves), `unproved` = the bench's deletion and insertion templates only.
--route-report repeats the steps with C2B_NO_ROUTE=1 and prints both kernel tables and the routing test's false-narrow reads
(kept for the narrow tier, failed there) and false-wide reads (sent to the wide ring, would have passed the narrow tier).
--one-kernel times the batches that launch the general kernel alone, one table per case: `coding1` = the bench amplicon with
a coding sequence, `coding3` = the bench's three HDR-mode amplicons and reads with a coding sequence on the first, `amp8` =
the bench amplicon and seven one-SNP alleles of it, `nosplit` = the bench batch under C2B_NO_SPLIT.
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


def one_kernel_case(case, n):
    """-> (workload, launch switch to set or None) of a --one-kernel case: batches that launch the general kernel alone"""
    from bench import Workload
    from crispresso2_b200 import synth
    w = Workload("hdr" if case == "coding3" else "single", n, 0)
    if case in ("coding1", "coding3"):           # a coding sequence on the first amplicon: split_all is false
        name = w.ref_names[0]
        w.refs[name] = dict(w.refs[name], contains_coding_seq=True, exon_positions=list(range(40, 200)), splicing_positions=[],
                            exon_len_mods=[0])
        return w, None
    if case == "amp8":                           # more than RG_MAX_REFS amplicons
        amp = w.refs["Reference"]["sequence"]
        for k in range(7):
            p = 30 + 30 * k
            w.refs["SNP%d" % k] = synth.amplicon_setup(amp[:p] + ("A" if amp[p] != "A" else "C") + amp[p + 1:])
            w.ref_names.append("SNP%d" % k)
        return w, None
    if case == "nosplit":
        return w, "C2B_NO_SPLIT"
    raise SystemExit("kernel_times: unknown --one-kernel case %r" % case)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reads", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mix", default="bench", choices=["bench", "proved", "unproved"])
    ap.add_argument("--json", help="also write the table as JSON here")
    ap.add_argument("--route-report", action="store_true",
                    help="also run the steps with C2B_NO_ROUTE=1 and report the diagonal tier's false-narrow / false-wide routing")
    ap.add_argument("--one-kernel", metavar="CASES",
                    help="time the general kernel alone instead, for each of these comma-separated cases: coding1, coding3, amp8, nosplit")
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
    eng = Engine(0)
    L = eng.L

    def load(w):
        """configure the engine for workload w and place its reads and outputs on the device -> one step"""
        P = w.params
        eng.configure(w.refs, w.ref_names, O.make_matrix(), P.needleman_wunsch_gap_open, P.needleman_wunsch_gap_extend,
                      P.aln_seed_count, P.aln_seed_min, w.flags, "ACGTN", 12)
        W = eng.string_width(w.max_len)
        R = len(w.ref_names)
        d_reads = torch.from_numpy(np.ascontiguousarray(w.buf)).to(dev)
        d_off = torch.from_numpy(w.off).to(dev)
        d_recs = torch.empty(n * 16, dtype=torch.uint8, device=dev)
        d_alns = torch.empty(n * R * 32, dtype=torch.uint8, device=dev)
        d_str = torch.empty(n * R * 2 * W, dtype=torch.uint8, device=dev)
        d_ed = torch.empty(n * R * 12 * 8, dtype=torch.uint8, device=dev)

        def step():
            rc = L.c2b_align_batch_device(eng.h, d_reads.data_ptr(), d_off.data_ptr(), n, w.max_len, None, None, None,
                                          d_recs.data_ptr(), d_alns.data_ptr(), d_str.data_ptr(), d_ed.data_ptr())
            if rc != 0:
                raise RuntimeError(L.c2b_last_error(eng.h).decode())
        return step

    def measure(step):
        """-> (per-launch rows, sum, diag counts per step, route counts per step) of args.steps profiled steps"""
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
        diag = route = None
        import ctypes as C
        if hasattr(L, "c2b_diag_counts"):
            a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
            if L.c2b_diag_counts(eng.h, C.byref(a), C.byref(b), C.byref(c)) == 0:
                diag = {"proved": a.value // args.steps, "tier1": b.value // args.steps, "tier2": c.value // args.steps}
        if hasattr(L, "c2b_route_counts"):
            a, b = C.c_int64(), C.c_int64()
            if L.c2b_route_counts(eng.h, C.byref(a), C.byref(b)) == 0:
                route = {"routed": a.value // args.steps, "kept": b.value // args.steps}
        return rows, total, diag, route

    def table(rows, total):
        print("| # | kernel | ms / launch | share |")
        print("|---|---|---|---|")
        for r in rows:
            print("| %d | %s | %.3f | %.0f %% |" % (r["launch"], r["kernel"], r["ms_per_launch"], 100.0 * r["ms_per_launch"] / total if total else 0.0))
        print("| | sum of kernel times per step | %.3f | |" % total)

    info = card_info(0)
    if args.one_kernel:
        cases = []
        for case in args.one_kernel.split(","):
            w, switch = one_kernel_case(case, n)
            step = load(w)
            if switch:
                os.environ[switch] = "1"
            try:
                rows, total, _, _ = measure(step)
            finally:
                if switch:
                    os.environ.pop(switch, None)
            if len(rows) != 1:
                raise SystemExit("kernel_times: --one-kernel %s launched %d kernels per step" % (case, len(rows)))
            print("card: %s, power limit %s W; --one-kernel %s: %d reads x 250 bp, %d amplicons, %d profiled steps after %d warm-up "
                  "steps" % (info.get("name"), info.get("power_limit_w"), case, n, len(w.ref_names), args.steps, args.warmup))
            table(rows, total)
            cases.append({"case": case, "amplicons": len(w.ref_names), "kernels": rows, "total_ms_per_step": total})
        if args.json:
            with open(args.json, "w") as fh:
                json.dump({"card": info, "reads": n, "steps": args.steps, "one_kernel": cases}, fh, indent=1)
        return
    w = Workload("single", n, 0)
    if args.mix != "bench":
        w.buf = mix_reads(args.mix, w.refs["Reference"], n).reshape(-1)
    step = load(w)
    rows, total, diag, route = measure(step)
    report = None
    if args.route_report:
        # the same steps without routing: whether a read passes the narrow tier depends on the read alone, so the narrow
        # failures without routing (N0), the routed reads (N_r) and the narrow failures with routing (N_f) give
        # false-narrow = N_f (kept, then failed) and false-wide = N_r - (N0 - N_f) (routed, would have passed)
        os.environ["C2B_NO_ROUTE"] = "1"
        try:
            rows0, total0, diag0, _ = measure(step)
        finally:
            os.environ.pop("C2B_NO_ROUTE", None)
        N0, Nr = diag0["tier2"], route["routed"]
        Nf = diag["tier2"] - Nr                          # tier-2 reads = routed + narrow failures
        report = {"listed": diag["tier1"], "N0": N0, "N_r": Nr, "N_f": Nf, "false_narrow": Nf, "false_wide": Nr - (N0 - Nf),
                  "kernels_no_route": rows0, "total_ms_no_route": total0}
    print("card: %s, power limit %s W, max SM clock %s MHz" % (info.get("name"), info.get("power_limit_w"), info.get("max_sm_clock_mhz")))
    print("%d reads x 250 bp (mix %s), %d profiled steps after %d warm-up steps; C2B_NO_DIAG=%s" % (
        n, args.mix, args.steps, args.warmup, os.environ.get("C2B_NO_DIAG", "")))
    table(rows, total)
    if diag is not None:
        print("reads per step: %d proved on the diagonal (%.1f %%), %d to the narrow tier, %d to the wide ring" %
              (diag["proved"], 100.0 * diag["proved"] / n, diag["tier1"], diag["tier2"]))
    if route is not None:
        print("routing per step: %d of the diagonal tier's unproved reads sent straight to the wide ring, %d kept for the narrow tier" %
              (route["routed"], route["kept"]))
    if report is not None:
        print("\nsame steps with C2B_NO_ROUTE=1:")
        table(report["kernels_no_route"], report["total_ms_no_route"])
        L_ = max(report["listed"], 1)
        print("routing report per step: listed %d, narrow failures without routing N0 = %d, routed N_r = %d, narrow failures with "
              "routing N_f = %d; false-narrow %d (%.2f %% of listed), false-wide %d (%.2f %% of listed)" % (
                  report["listed"], report["N0"], report["N_r"], report["N_f"], report["false_narrow"],
                  100.0 * report["false_narrow"] / L_, report["false_wide"], 100.0 * report["false_wide"] / L_))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": info, "reads": n, "steps": args.steps, "mix": args.mix, "no_diag": os.environ.get("C2B_NO_DIAG", ""),
                       "kernels": rows, "total_ms_per_step": total, "diag_counts": diag, "route_counts": route,
                       "route_report": report}, fh, indent=1)


if __name__ == "__main__":
    main()
