"""One forward plus one backward pass of odeint_adjoint with adjoint_options={'fused_vjp': True}: the shared step (the
default) against independent rows (options={'independent_rows': True}, k_rows_adaptive forward, k_rows_adjoint backward).

Lorenz 65 536 x 3 fp64 (config 2's system and inputs) and the same at 1 048 576 rows, where the shared step runs on the
stage kernels: dopri5, y0 = 1 + 0.1 randn (default_rng(0)), t = arange(11) * 0.01, odeint_adjoint's default tolerances, the
loss a fixed random weighting of the solution.  Each workload warms both arms up, then alternates them `--runs` times; each
run is timed with CUDA events around forward + backward, ending in a synchronise.  Prints the GPU, its power limit and
maximum SM clock, and one JSON line per workload: median and all times, both arms' backward attempts, and the spread of the
per-row backward attempts (min / median / max) of the independent-rows arm.

    python scripts/rows_adjoint_bench.py [--runs 5]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import tfdiffeq_b200 as tfd  # noqa: E402
from adjoint_bench import gpu_info  # noqa: E402


def workload(n):
    rng = np.random.default_rng(0)
    y0 = torch.tensor(1.0 + 0.1 * rng.standard_normal((n, 3)), device="cuda")
    t = torch.tensor(np.arange(11) * 0.01, device="cuda")
    w = torch.tensor(np.random.default_rng(1).standard_normal((11, n, 3)), device="cuda")
    return "lorenz_%dx3_f64_dopri5" % n, tfd.rhs.Lorenz(), y0, t, w


def step(mod, y0, t, w, rows):
    y = y0.clone().requires_grad_(True)
    opts = {"fused_vjp": True}
    if rows:
        opts["independent_rows"] = True
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    sol = tfd.odeint_adjoint(mod, y, t, method="dopri5", options=opts)
    (sol * w).sum().backward()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end), y.grad, tfd.adjoint.last_stats["backward"]


def compare(wl, runs):
    name, mod, y0, t, w = wl
    arms = ("shared_step", "independent_rows")
    for arm in arms:                                          # warm-up
        step(mod, y0, t, w, arm == "independent_rows")
    times = {arm: [] for arm in arms}
    res = {}
    for _ in range(runs):
        for arm in arms:
            ms, g, back = step(mod, y0, t, w, arm == "independent_rows")
            times[arm].append(ms)
            res[arm] = (g, back)
    out = dict(workload=name, runs=runs)
    for arm in arms:
        out[arm + "_ms"] = float(np.median(times[arm]))
        out[arm + "_ms_all"] = [round(x, 3) for x in times[arm]]
    out["shared_step_backward_attempts"] = sum(b["n_accepted"] + b["n_rejected"] for b in res["shared_step"][1])
    rb = res["independent_rows"][1]
    att = (rb["row_accepted"] + rb["row_rejected"]).cpu().numpy()
    out["independent_rows_backward_attempts"] = int(att.sum())
    out["row_backward_attempts_min_median_max"] = [int(att.min()), float(np.median(att)), int(att.max())]
    out["speedup"] = out["shared_step_ms"] / out["independent_rows_ms"]
    g0, g1 = res["shared_step"][0], res["independent_rows"][0]
    out["max_rel_grad_diff"] = float((g1 - g0).abs().max()) / max(float(g0.abs().max()), 1e-300)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rows_adjoint_bench.py needs a GPU")
    print(json.dumps(gpu_info()), flush=True)
    for n in (65536, 1048576):
        print(json.dumps(compare(workload(n), max(a.runs, 5))), flush=True)
    print(json.dumps(gpu_info()), flush=True)


if __name__ == "__main__":
    main()
