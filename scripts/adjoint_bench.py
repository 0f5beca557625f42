"""One forward plus one backward pass of odeint_adjoint, with the backward's augmented dynamics from torch autograd (the
default) and from the stage kernels (adjoint_options={'fused_vjp': True}).

(a) Lorenz, config 2's system and inputs over a short horizon: 65 536 x 3 fp64, dopri5, y0 = 1 + 0.1 randn
    (default_rng(0)), t = arange(11) * 0.01, odeint_adjoint's default tolerances;
(b) CubicMLP(50), ode_demo's network: 131 072 x 2 fp32, dopri5, initial states along ode_demo's spiral, t = linspace(0, 0.5, 6).

The loss is a fixed random weighting of the solution.  Each workload warms both arms up, then alternates them `--runs` times;
each run is timed with CUDA events around forward + backward, ending in a synchronise.  Prints the GPU, its power limit and
maximum SM clock, and one JSON line per workload: median and all times, the backward NFE and the attempts of every backward
interval for both arms, and the largest relative difference of the gradients between the arms.

    python scripts/adjoint_bench.py [--runs 5]
"""
import argparse
import json
import os
import subprocess
import sys

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


def lorenz_workload():
    rng = np.random.default_rng(0)
    y0 = torch.tensor(1.0 + 0.1 * rng.standard_normal((65536, 3)), device="cuda")
    t = torch.tensor(np.arange(11) * 0.01, device="cuda")
    w = torch.tensor(np.random.default_rng(1).standard_normal((11, 65536, 3)), device="cuda")
    return "lorenz_65536x3_f64_dopri5", tfd.rhs.Lorenz(), y0, t, w


def cubic_mlp_workload():
    n = 131072
    rng = np.random.default_rng(0)
    th = rng.uniform(0.0, 6.0, n)
    r = 2.0 * np.exp(-th / 4.0) * (1.0 + 0.05 * rng.standard_normal(n))
    y0 = torch.tensor(np.stack([r * np.cos(th), r * np.sin(th)], 1), dtype=torch.float32, device="cuda")
    t = torch.linspace(0.0, 0.5, 6, device="cuda")
    w = torch.tensor(np.random.default_rng(1).standard_normal((6, n, 2)), dtype=torch.float32, device="cuda")
    mod = tfd.rhs.CubicMLP(50, generator=torch.Generator().manual_seed(0)).cuda()
    return "cubic_mlp50_131072x2_f32_dopri5", mod, y0, t, w


def step(mod, y0, t, w, fused):
    y = y0.clone().requires_grad_(True)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    sol = tfd.odeint_adjoint(mod, y, t, method="dopri5", adjoint_options={"fused_vjp": True} if fused else None)
    (sol * w).sum().backward()
    end.record()
    torch.cuda.synchronize()
    grads = [y.grad] + [p.grad.clone() for p in mod.parameters() if p.grad is not None]
    for p in mod.parameters():
        p.grad = None
    back = tfd.adjoint.last_stats["backward"]
    return start.elapsed_time(end), grads, back


def compare(workload, runs):
    name, mod, y0, t, w = workload
    arms = ("autograd", "fused_vjp")
    for arm in arms:                                          # warm-up
        step(mod, y0, t, w, arm == "fused_vjp")
    times = {arm: [] for arm in arms}
    res = {}
    for _ in range(runs):
        for arm in arms:
            ms, grads, back = step(mod, y0, t, w, arm == "fused_vjp")
            times[arm].append(ms)
            res[arm] = (grads, back)
    out = dict(workload=name, runs=runs)
    for arm in arms:
        back = res[arm][1]
        out[arm + "_ms"] = float(np.median(times[arm]))
        out[arm + "_ms_all"] = [round(x, 3) for x in times[arm]]
        out[arm + "_backward_nfe"] = sum(b["nfe"] for b in back)
        out[arm + "_attempts_per_interval"] = [b["n_accepted"] + b["n_rejected"] for b in back]
    out["speedup"] = out["autograd_ms"] / out["fused_vjp_ms"]
    out["nfe_match"] = out["autograd_backward_nfe"] == out["fused_vjp_backward_nfe"]
    out["max_rel_grad_diff"] = max(float((a - b).abs().max()) / max(float(b.abs().max()), 1e-300)
                                   for a, b in zip(res["fused_vjp"][0], res["autograd"][0]))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adjoint_bench.py needs a GPU")
    print(json.dumps(gpu_info()), flush=True)
    for wl in (lorenz_workload, cubic_mlp_workload):
        print(json.dumps(compare(wl(), max(a.runs, 3))), flush=True)
    print(json.dumps(gpu_info()), flush=True)


if __name__ == "__main__":
    main()
