"""One forward plus one backward pass through odeint(options={'backprop': True}) against odeint_adjoint with
adjoint_options={'fused_vjp': True}, on the two workloads of scripts/adjoint_bench.py:

(a) Lorenz 65 536 x 3 fp64, dopri5, 11 outputs;
(b) CubicMLP(50) 131 072 x 2 fp32, dopri5, 6 outputs.

Each arm is warmed up, then the arms alternate `--runs` times, each run timed with CUDA events around forward + backward
and ending in a synchronise; the peak device memory of each arm is taken from a run of its own after a reset.  Prints the
GPU, its power limit and maximum SM clock, and one JSON line per workload: median and all times, peak memory, the forward
step counts and the largest relative difference of the gradients between the arms (discretise-then-optimise against
optimise-then-discretise: expected at the solver tolerance, not at rounding).

    python scripts/backprop_bench.py [--runs 5]
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
from adjoint_bench import cubic_mlp_workload, gpu_info, lorenz_workload  # noqa: E402


def step(mod, y0, t, w, arm):
    y = y0.clone().requires_grad_(True)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    if arm == "backprop":
        sol = tfd.odeint(mod, y, t, method="dopri5", options={"backprop": True})
    else:
        sol = tfd.odeint_adjoint(mod, y, t, method="dopri5", adjoint_options={"fused_vjp": True})
    steps = tfd.solvers.last_stats["n_accepted"] if arm == "backprop" else None
    (sol * w).sum().backward()
    end.record()
    torch.cuda.synchronize()
    grads = [y.grad] + [p.grad.clone() for p in mod.parameters() if p.grad is not None]
    for p in mod.parameters():
        p.grad = None
    return start.elapsed_time(end), grads, steps


def compare(workload, runs):
    name, mod, y0, t, w = workload
    arms = ("backprop", "adjoint_fused_vjp")
    out = dict(workload=name, runs=runs)
    for arm in arms:
        step(mod, y0, t, w, arm)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step(mod, y0, t, w, arm)
        out[arm + "_peak_mib"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    times = {arm: [] for arm in arms}
    res = {}
    for _ in range(runs):
        for arm in arms:
            ms, grads, steps = step(mod, y0, t, w, arm)
            times[arm].append(ms)
            res[arm] = grads
            if steps is not None:
                out["forward_steps"] = steps
    for arm in arms:
        out[arm + "_ms"] = float(np.median(times[arm]))
        out[arm + "_ms_all"] = [round(x, 3) for x in times[arm]]
    out["max_rel_grad_diff"] = max(float((a - b).abs().max()) / max(float(b.abs().max()), 1e-300)
                                   for a, b in zip(res["backprop"], res["adjoint_fused_vjp"]))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("backprop_bench.py needs a GPU")
    print(json.dumps(gpu_info()), flush=True)
    for wl in (lorenz_workload, cubic_mlp_workload):
        print(json.dumps(compare(wl(), max(a.runs, 3))), flush=True)
    print(json.dumps(gpu_info()), flush=True)


if __name__ == "__main__":
    main()
