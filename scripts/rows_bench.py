"""Shared step against independent rows (options={'independent_rows': True}) on the benchmark's Lorenz system.

(a) config 2's system and inputs: 65 536 x 3 fp64, dopri5, y0 = 1 + 0.1 randn (default_rng(0)), t = arange(1000) * 0.01,
    default tolerances -- the shared step runs in the persistent kernel;
(b) the same system at 1 048 576 rows -- beyond the persistent kernel's capacity, the shared step takes the stage kernels.

Each comparison warms both arms up, then alternates them `--runs` times; every run is timed with a host clock around a solve
that ends in a synchronise.  Prints the GPU, its power limit and maximum SM clock, and one JSON line per comparison: median
times, the per-row accepted-step distribution against the shared solve's count, and row-steps per second (accepted steps
summed over rows, over the median time).

    python scripts/rows_bench.py [--runs 5] [--sizes 65536,1048576]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tfdiffeq_b200 as tfd  # noqa: E402


def gpu_info():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [x.strip() for x in q.split(",")]
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        info["power_limit"] = info["max_sm_clock"] = "unavailable (%s)" % e
    return info


def solve(y0, t, rows):
    opts = {"independent_rows": True} if rows else None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)      # the shared step's fall-back to the stage kernels at 1 M rows
        sol = tfd.odeint(tfd.rhs.Lorenz(), y0, t, method="dopri5", options=opts)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, sol, dict(tfd.last_stats)


def compare(n, runs):
    rng = np.random.default_rng(0)
    y0 = torch.tensor(1.0 + 0.1 * rng.standard_normal((n, 3)), device="cuda")
    t = torch.tensor(np.arange(1000) * 0.01)
    times = {"shared": [], "rows": []}
    stats = {}
    for arm in ("shared", "rows"):                           # warm-up
        solve(y0, t, arm == "rows")
    for _ in range(runs):
        for arm in ("shared", "rows"):
            dt, sol, st = solve(y0, t, arm == "rows")
            times[arm].append(dt)
            stats[arm] = st
            del sol
    sh, ro = stats["shared"], stats["rows"]
    acc = ro["row_accepted"].cpu().numpy()
    med = {arm: float(np.median(v)) for arm, v in times.items()}
    return dict(
        rows=n, runs=runs,
        shared_path="persistent kernel" if sh["fused_rhs"] else "stage kernels",
        shared_ms=med["shared"] * 1e3, rows_ms=med["rows"] * 1e3, rows_over_shared=med["rows"] / med["shared"],
        shared_ms_all=[round(x * 1e3, 3) for x in times["shared"]], rows_ms_all=[round(x * 1e3, 3) for x in times["rows"]],
        shared_accepted=sh["n_accepted"], shared_rejected=sh["n_rejected"],
        row_accepted_min=int(acc.min()), row_accepted_median=float(np.median(acc)), row_accepted_max=int(acc.max()),
        row_rejected_total=ro["n_rejected"],
        shared_row_steps_per_s=sh["n_accepted"] * n / med["shared"], rows_row_steps_per_s=float(acc.sum()) / med["rows"])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--sizes", default="65536,1048576")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rows_bench.py needs a GPU")
    print(json.dumps(gpu_info()), flush=True)
    for n in (int(x) for x in a.sizes.split(",")):
        print(json.dumps(compare(n, max(a.runs, 3))), flush=True)


if __name__ == "__main__":
    main()
