"""Time ws_metrics_eval (csrc/ws_metrics.cu) stage by stage: the key / histogram pass, each of the eight radix passes and
the evaluation, with CUDA events recorded between the stages by the entry point itself; bytes each stage must move over its
time as a share of the H100 SXM data-sheet 3.35 TB/s; and, for scale, the numpy oracle (stable argsort, curves, EER, one
minDCF) on the host over the same arrays.

Workload: 5-decimal scores (what score files carry, so ties are common) of 10 % target trials at the sizes of a VoxCeleb1-O
list (37 720), VoxCeleb1-H (579 818) and two synthetic large lists (10^7, 10^8).  The card's name and power limit are read
in the same run.  Usage: python tools/metrics_bench.py [--sizes ...] [--reps R] [--out file.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import metrics_np  # noqa: E402
from wespeaker_b200 import metrics  # noqa: E402

PEAK_BPS = 3.35e12
STAGES = ["keys"] + [f"pass{p}" for p in range(8)] + ["eval"]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def active_passes(s: np.ndarray):
    """Which 8-bit digits of the order keys differ between trials (the passes the sort runs)."""
    b = (s + 0.0).view(np.uint64)
    k = np.where(b >> np.uint64(63), ~b, b | np.uint64(1 << 63))
    return [bool((((k >> np.uint64(8 * p)) & np.uint64(255)) != ((k[0] >> np.uint64(8 * p)) & np.uint64(255))).any())
            for p in range(8)]


def stage_bytes(n, active):
    return {"keys": 21 * n, **{f"pass{p}": (32 * n if a else 0) for p, a in enumerate(active)}, "eval": 8 * n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="*", default=[37720, 579818, 10_000_000, 100_000_000])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--oracle-max", type=int, default=100_000_000, help="largest n the host oracle is timed at")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("metrics_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    results = {"card": card(), "rows": []}
    pts = [(0.01, 1, 1)]
    for n in a.sizes:
        rng = np.random.default_rng(n)
        lab = rng.random(n) < 0.1
        s = np.round(0.25 * rng.standard_normal(n) + 0.5 * lab, 5)
        active = active_passes(s)
        sd = torch.from_numpy(s).to(dev)
        ld = torch.from_numpy(lab).to(dev).to(torch.uint8)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
        for e in ev:
            e.record()                       # creates the underlying event
        times = {k: [] for k in STAGES + ["total"]}
        for rep in range(3 + a.reps):
            out = metrics._launch(sd, ld, pts, stage_events=ev)
            torch.cuda.synchronize()
            assert int(out[7].item()) == 0
            if rep >= 3:
                for i, k in enumerate(STAGES):
                    times[k].append(ev[i].elapsed_time(ev[i + 1]))
                times["total"].append(ev[0].elapsed_time(ev[-1]))
        med = {k: float(np.median(v)) for k, v in times.items()}
        by = stage_bytes(n, active)
        row = {"n": n, "active_passes": sum(active), "ms": med,
               "hbm_share": {k: (by[k] / (med[k] * 1e-3) / PEAK_BPS if by[k] else None) for k in STAGES},
               "trials_per_s": n / (med["total"] * 1e-3)}
        metrics.evaluate(sd, ld, pts)
        t0 = time.perf_counter()
        m = metrics.evaluate(sd, ld, pts)
        row["evaluate_call_ms"] = (time.perf_counter() - t0) * 1e3
        if n <= a.oracle_max:
            t0 = time.perf_counter()
            fnr, fpr = metrics_np.pmiss_pfa_rbst(s, lab)
            eer, thr = metrics_np.eer(fnr, fpr, s)
            mdcf = metrics_np.c_norm(fnr, fpr, 0.01)
            row["oracle_numpy_ms"] = (time.perf_counter() - t0) * 1e3
            row["bit_equal_to_oracle"] = bool(eer == m.eer and thr == m.threshold and mdcf == m.min_dcf[0])
        results["rows"].append(row)
        print(json.dumps(row), flush=True)
        del sd, ld
        torch.cuda.empty_cache()
    print(json.dumps({"card": results["card"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
