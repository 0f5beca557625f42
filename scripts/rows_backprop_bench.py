"""One forward plus one backward pass of odeint(..., options={'backprop': True}) with independent rows
(options={'independent_rows': True}: k_rows_adaptive's recording forward, one k_rows_bp launch backward) against

* the per-row continuous adjoint (odeint_adjoint with independent_rows and fused_vjp) and the shared-step backprop path,
  on Lorenz 65 536 x 3 and 1 048 576 x 3 fp64 dopri5 (y0 = 1 + 0.1 randn (default_rng(0)), t = arange(11) * 0.01,
  odeint's default tolerances);
* the shared-step backprop path on a trainable CubicMLP(50) with 131 072 x 2 fp32 rows (y0 = 0.5 randn, t = linspace(0, 1,
  11), rtol 1e-4, atol 1e-6).

The loss is a fixed random weighting of the solution.  Each workload warms every arm up, then alternates the arms `--runs`
times (at least 5); each run is timed with CUDA events around forward + backward, ending in a synchronise, and the peak
device memory of the run is read with torch.cuda.max_memory_allocated.  Prints the GPU, its power limit and maximum SM clock
before and after, and one JSON line per workload: median and all times and the peak memory of every arm, the per-row
backprop's re-run flag and steps, and the largest relative y0-gradient difference from the shared-step backprop arm.

    python scripts/rows_backprop_bench.py [--runs 5]
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


def lorenz(n):
    rng = np.random.default_rng(0)
    y0 = torch.tensor(1.0 + 0.1 * rng.standard_normal((n, 3)), device="cuda")
    t = torch.tensor(np.arange(11) * 0.01, device="cuda")
    w = torch.tensor(np.random.default_rng(1).standard_normal((11, n, 3)), device="cuda")
    return "lorenz_%dx3_f64_dopri5" % n, tfd.rhs.Lorenz(), y0, t, w, {}, ("rows_backprop", "rows_adjoint", "shared_backprop")


def cubic(n):
    g = torch.Generator().manual_seed(0)
    mod = tfd.rhs.CubicMLP(50, dtype=torch.float32, generator=g).cuda()
    y0 = (0.5 * torch.randn(n, 2, generator=g)).cuda()
    t = torch.linspace(0, 1, 11, dtype=torch.float64)
    w = torch.randn((11, n, 2), generator=g).cuda()
    return ("cubic_mlp50_%dx2_f32_dopri5_trainable" % n, mod, y0, t, w, dict(rtol=1e-4, atol=1e-6),
            ("rows_backprop", "shared_backprop"))


def step(mod, y0, t, w, arm, tol):
    y = y0.clone().requires_grad_(True)
    for p in mod.parameters():
        p.grad = None
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    start.record()
    if arm == "rows_adjoint":
        sol = tfd.odeint_adjoint(mod, y, t, method="dopri5", options={"independent_rows": True, "fused_vjp": True}, **tol)
    else:
        opts = {"backprop": True}
        if arm == "rows_backprop":
            opts["independent_rows"] = True
        sol = tfd.odeint(mod, y, t, method="dopri5", options=opts, **tol)
    (sol * w).sum().backward()
    end.record()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    stats = dict(tfd.backprop.last_stats) if arm == "rows_backprop" else {}
    return start.elapsed_time(end), peak, y.grad, stats


def compare(wl, runs):
    name, mod, y0, t, w, tol, arms = wl
    for arm in arms:                                          # warm-up
        step(mod, y0, t, w, arm, tol)
    times = {arm: [] for arm in arms}
    peaks, grads, stats = {}, {}, {}
    for _ in range(runs):
        for arm in arms:
            ms, peak, g, st = step(mod, y0, t, w, arm, tol)
            times[arm].append(ms)
            peaks[arm], grads[arm] = peak, g
            if st:
                stats = st
    out = dict(workload=name, runs=runs)
    for arm in arms:
        out[arm + "_ms"] = float(np.median(times[arm]))
        out[arm + "_ms_all"] = [round(x, 3) for x in times[arm]]
        out[arm + "_peak_mib"] = round(peaks[arm] / 2 ** 20, 1)
    out["rows_backprop_steps"] = stats.get("steps")
    out["rows_backprop_rerun"] = stats.get("rerun")
    g0, g1 = grads["shared_backprop"], grads["rows_backprop"]
    out["max_rel_grad_diff_vs_shared_backprop"] = float((g1 - g0).abs().max()) / max(float(g0.abs().max()), 1e-300)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rows_backprop_bench.py needs a GPU")
    print(json.dumps(gpu_info()), flush=True)
    for wl in (lorenz(65536), lorenz(1048576), cubic(131072)):
        print(json.dumps(compare(wl, max(a.runs, 5))), flush=True)
    print(json.dumps(gpu_info()), flush=True)


if __name__ == "__main__":
    main()
