"""examples/latent_ode.py's training step through the solve: LatentODEFunc (4 -> 20 -> 20 -> 4, ELU) as a built-in
right-hand side against the same network as a plain torch module.

* Training step, forward plus backward: z0 = 1000 x 4 (randn, seed 0), the first 100 times of generate_spiral2d's grid
  (linspace(0, 6 pi, 1000)), dopri5, rtol 1e-7, atol 1e-9, trainable weights, loss (pred * w).sum() with a fixed random
  w.  Arms, for fp32 and fp64:
    - ``backprop``: odeint(..., options={'backprop': True}) on the built-in (k_bp_rhs, no forward or autograd call);
    - ``torch``: the same with fused_rhs=False, i.e. the module's forward and autograd on the generic path, equal weights;
    - ``fused_vjp``: odeint_adjoint with adjoint_options={'fused_vjp': True}.
* Forward solve alone, 65 536 rows, same times and method, frozen weights: the persistent kernel (``fused``),
  ``independent_rows`` and the torch module (fused_rhs=False).

Each workload warms every arm up, then alternates the arms `--runs` times (at least 5); each run is timed with CUDA
events, ending in a synchronise, and its peak device memory is read with torch.cuda.max_memory_allocated.  Prints the GPU,
its power limit and maximum SM clock before and after, and one JSON line per workload: median and all times, peak memory,
and each arm's largest relative difference from the torch arm (y0 and parameter gradients, or the solution).

    python scripts/latent_bench.py [--runs 5]
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

TOL = dict(rtol=1e-7, atol=1e-9, method="dopri5")


def samp_ts(dtype):
    return torch.linspace(0.0, 6.0 * np.pi, 1000, dtype=dtype)[:100].cuda()


def module(dtype, trainable):
    mod = tfd.rhs.LatentODEFunc(4, 20, dtype=dtype, generator=torch.Generator().manual_seed(1)).cuda()
    for p in mod.parameters():
        p.requires_grad_(trainable)
    return mod


def train_step(mod, z0, t, w, arm):
    y = z0.clone().requires_grad_(True)
    for p in mod.parameters():
        p.grad = None
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    start.record()
    if arm == "fused_vjp":
        pred = tfd.odeint_adjoint(mod, y, t, adjoint_options={"fused_vjp": True}, **TOL)
    else:
        opts = {"backprop": True} if arm == "backprop" else {"backprop": True, "fused_rhs": False}
        pred = tfd.odeint(mod, y, t, options=opts, **TOL)
    (pred * w).sum().backward()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end), torch.cuda.max_memory_allocated() - base, [y.grad] + [p.grad for p in mod.parameters()]


def forward_solve(mod, z0, t, arm):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    opts = {"fused": None, "rows": {"independent_rows": True}, "torch": {"fused_rhs": False}}[arm]
    start.record()
    sol = tfd.odeint(mod, z0, t, options=opts, **TOL)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end), torch.cuda.max_memory_allocated() - base, [sol]


def rel(a, b):
    return max(float((x - z).abs().max()) / max(float(z.abs().max()), 1e-300) for x, z in zip(a, b))


def compare(name, arms, run, runs):
    for arm in arms:
        run(arm)
    times = {arm: [] for arm in arms}
    peaks, outs = {}, {}
    for _ in range(runs):
        for arm in arms:
            ms, peak, out = run(arm)
            times[arm].append(ms)
            peaks[arm], outs[arm] = peak, out
    res = dict(workload=name, runs=runs)
    for arm in arms:
        res[arm + "_ms"] = round(float(np.median(times[arm])), 3)
        res[arm + "_ms_all"] = [round(x, 3) for x in times[arm]]
        res[arm + "_peak_mib"] = round(peaks[arm] / 2 ** 20, 1)
        if arm != "torch":
            res[arm + "_max_rel_diff_vs_torch"] = rel(outs[arm], outs["torch"])
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("latent_bench.py needs a GPU")
    runs = max(a.runs, 5)
    print(json.dumps(gpu_info()), flush=True)
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        g = torch.Generator().manual_seed(0)
        z0 = torch.randn(1000, 4, dtype=dtype, generator=g).cuda()
        w = torch.randn(100, 1000, 4, dtype=dtype, generator=g).cuda()
        mod, t = module(dtype, True), samp_ts(dtype)
        print(json.dumps(compare("latent_train_1000x4_%s_dopri5" % tag, ("backprop", "torch", "fused_vjp"),
                                 lambda arm: train_step(mod, z0, t, w, arm), runs)), flush=True)
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        z0 = torch.randn(65536, 4, dtype=dtype, generator=torch.Generator().manual_seed(0)).cuda()
        mod, t = module(dtype, False), samp_ts(dtype)
        print(json.dumps(compare("latent_forward_65536x4_%s_dopri5" % tag, ("fused", "rows", "torch"),
                                 lambda arm: forward_solve(mod, z0, t, arm), runs)), flush=True)
    print(json.dumps(gpu_info()), flush=True)


if __name__ == "__main__":
    main()
