"""The linear right-hand side y' = y @ A (rhs.LinearODE) at the north-star size, 65 536 x 128 fp64.

(a) One evaluation, CUDA events around every launch, L2 flushed before each:
      linear_nk0          b2ode_linear_f64, plain product                        reads Y, writes out
      linear_nk5          b2ode_linear_f64 fed by dopri5 stage 4's combine       reads y0 + 5 k, writes out
      linear_nk5_ystage   the same, also storing the stage input (the last stage stores y1)
      dgemm               torch.matmul (cuBLAS DGEMM)                            reads Y, writes out
      stage5_dgemm        k_rk_stage (dopri5 stage 4, 5 terms) + DGEMM           the unfused stage: y_i goes through HBM
    Algorithmic bytes and FLOPs come from the shapes; the share of peak is the larger of bytes / 3.35 TB/s and
    FLOPs / 67 TFLOP/s (H100 SXM data sheet) over the measured time, with the bound named.
(b) The north-star solve (bench.py's `northstar`: BatchedLinear(dim=128, seed=0), y0 from seed 100, t = linspace(0, 2, 11),
    dopri5, rtol 1e-6, atol 1e-9) with LinearODE against the external BatchedLinear func, eager and with cuda_graph, plus
    LinearODE with fused_rhs=False; arms alternate, three runs each, host clock around a solve that ends in a device
    synchronise.  Counts of every arm and the max |difference| between arms are recorded.

Usage: python scripts/linear_bench.py [--launches 200] [--out FILE.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import tfdiffeq_b200 as tfd                     # noqa: E402
from tfdiffeq_b200 import _lib, rhs, tableaus   # noqa: E402
from problems import PROBLEMS                   # noqa: E402

PEAK_BW, PEAK_F64 = 3.35e12, 67e12
M, D = 65536, 128


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit=power, clocks_max_sm=clock)
    except Exception as e:                      # the measurement still stands; say what is missing
        return dict(name=torch.cuda.get_device_name(), error="nvidia-smi query failed: %r" % (e,))


def time_launches(fn, flush, launches, warmup=10):
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(launches)]
    for i in range(launches):
        flush.fill_(i & 0xFF)
        ev[i][0].record()
        fn()
        ev[i][1].record()
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    return dict(median_ms=float(np.median(ms)), mean_ms=float(ms.mean()), min_ms=float(ms.min()), max_ms=float(ms.max()),
                launches=launches)


def roof(t_ms, nbytes, flops):
    s = t_ms * 1e-3
    tb, tf = nbytes / PEAK_BW, flops / PEAK_F64
    bound = "hbm" if tb >= tf else "fp64_tensor"
    return dict(bytes=int(nbytes), flops=int(flops), gb_per_s=nbytes / s / 1e9, gflop_per_s=flops / s / 1e9,
                bound=bound, share_of_bound=max(tb, tf) / s)


class StageKernel(object):
    """A dopri5 solver handle whose only use is launching k_rk_stage for one stage row (b2ode_rk_stage)."""

    def __init__(self, y0, ks, ystage, dt):
        tab = tableaus.DOPRI5
        lib = _lib.lib
        dev = y0.device
        d = _lib.AdaptiveDesc()
        d.dtype, d.nseg, d.n_k, d.fsal = _lib.F64, 1, tab.n_k, 1
        d.seg_len[0] = y0.numel()
        for i, row in enumerate(tab.beta):
            for j, v in enumerate(row):
                d.beta[i][j] = v
        for j in range(tab.n_k):
            d.c_sol[j], d.c_error[j], d.c_mid[j] = tab.c_sol[j], tab.c_error[j], tab.c_mid[j]
        d.sm_count = torch.cuda.get_device_properties(dev).multi_processor_count
        self.h = C.c_void_p()
        _lib.check(lib.b2ode_adaptive_create(C.byref(self.h), C.byref(d)))
        st = _lib.State()
        st.dt = dt
        self.state = torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(dev)
        self.ws = torch.empty(max(int(lib.b2ode_workspace_bytes(C.byref(d))), 32), dtype=torch.uint8, device=dev)
        self.tstage = torch.zeros(tab.n_k, dtype=torch.float64, device=dev)
        self.t_out = torch.zeros(1, dtype=torch.float64, device=dev)
        self.out = torch.empty_like(y0)
        b = _lib.AdaptiveBuffers()
        b.state, b.workspace, b.workspace_bytes = self.state.data_ptr(), self.ws.data_ptr(), self.ws.numel()
        b.y0[0], b.f0[0], b.ystage[0] = y0.data_ptr(), ks[0].data_ptr(), ystage.data_ptr()
        b.tstage, b.t_out, b.n_out, b.out[0] = self.tstage.data_ptr(), self.t_out.data_ptr(), 1, self.out.data_ptr()
        _lib.check(lib.b2ode_adaptive_bind(self.h, C.byref(b), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        self.kp = []
        for i in range(1, len(ks)):
            arr = _lib.PtrArray()
            arr[0] = ks[i].data_ptr()
            self.kp.append(arr)
            _lib.check(lib.b2ode_set_k(self.h, i, arr))

    def stage(self, row):
        _lib.check(_lib.lib.b2ode_rk_stage(self.h, row, self.kp[row - 1]))

    def close(self):
        _lib.lib.b2ode_adaptive_destroy(self.h)


def kernel_section(launches):
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)      # > H100's 50 MB L2
    g = torch.Generator(device=dev).manual_seed(0)
    A = torch.tensor(PROBLEMS["batched_linear"](backend="numpy", dim=D, seed=0).A, device=dev)
    y0 = torch.randn(M, D, dtype=torch.float64, device=dev, generator=g)
    ks = [torch.randn(M, D, dtype=torch.float64, device=dev, generator=g) for _ in range(5)]
    ys = torch.empty_like(y0)
    dt = 0.05
    row = 4                                         # dopri5 stage row 4: five nonzero terms
    coefs = list(tableaus.DOPRI5.beta[row])
    st = StageKernel(y0, ks, ys, dt)
    stage = (ks, coefs, st.state.data_ptr(), None)
    stage_ys = (ks, coefs, st.state.data_ptr(), ys)
    buf = M * D * 8
    flops = 2.0 * M * D * D
    res = {}
    arms = {
        "linear_nk0": (lambda: rhs.linear_f64(y0, A), 2 * buf, flops),
        "linear_nk5": (lambda: rhs.linear_f64(y0, A, stage=stage), 7 * buf, flops),
        "linear_nk5_ystage": (lambda: rhs.linear_f64(y0, A, stage=stage_ys), 8 * buf, flops),
        "dgemm": (lambda: torch.matmul(y0, A), 2 * buf, flops),
        "stage5_dgemm": (lambda: (st.stage(row), torch.matmul(ys, A)), 9 * buf, flops),
    }
    for name, (fn, nbytes, fl) in arms.items():
        r = time_launches(fn, flush, launches)
        r.update(roof(r["median_ms"], nbytes, fl))
        res[name] = r
        print("%-18s %8.4f ms  %7.1f GB/s  %7.1f GFLOP/s  %5.1f %% of the %s bound" % (
            name, r["median_ms"], r["gb_per_s"], r["gflop_per_s"], 100 * r["share_of_bound"], r["bound"]), flush=True)
    # the fused evaluation equals the unfused one bit for bit
    st.stage(row)
    fused = rhs.linear_f64(y0, A, stage=stage)
    res["fused_equals_stage_kernel_then_linear"] = bool(torch.equal(fused, rhs.linear_f64(ys, A)))
    res["max_abs_linear_vs_dgemm"] = float((rhs.linear_f64(y0, A) - torch.matmul(y0, A)).abs().max())
    torch.cuda.synchronize()
    st.close()
    return res


def solve_section(runs):
    dev = torch.device("cuda:0")
    f_np = PROBLEMS["batched_linear"](backend="numpy", dim=D, seed=0)
    ext = PROBLEMS["batched_linear"](backend="torch", device=dev, dim=D, seed=0)
    lin = rhs.LinearODE(f_np.A).to(dev)
    y0 = torch.tensor(np.random.default_rng(100).standard_normal((M, D)), device=dev)
    t = torch.tensor(np.linspace(0., 2., 11))
    arms = {
        "linear_eager": (lin, {}),
        "external_eager": (ext, {}),
        "linear_cuda_graph": (lin, {"cuda_graph": True}),
        "external_cuda_graph": (ext, {"cuda_graph": True}),
        "linear_unfused_eager": (lin, {"fused_rhs": False}),
    }
    times = {k: [] for k in arms}
    stats, sols = {}, {}
    for name, (f, opt) in arms.items():      # warm-up: module loads, cuBLAS heuristics, the image cache
        tfd.odeint(f, y0, t, rtol=1e-6, atol=1e-9, method="dopri5", options=opt)
    torch.cuda.synchronize()
    for _ in range(runs):
        for name, (f, opt) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sol = tfd.odeint(f, y0, t, rtol=1e-6, atol=1e-9, method="dopri5", options=opt)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)
            s = dict(tfd.last_stats)
            stats[name] = {k: s[k] for k in ("n_accepted", "n_rejected", "nfe", "stage_func", "cuda_graph")}
            sols[name] = sol
    res = {}
    for name in arms:
        ms = np.array(times[name])
        res[name] = dict(median_ms=float(np.median(ms)), min_ms=float(ms.min()), max_ms=float(ms.max()),
                         runs=[float(x) for x in ms], **stats[name])
        print("%-22s median %8.2f ms  (%.2f .. %.2f)  acc %d rej %d nfe %d stage_func %s" % (
            name, res[name]["median_ms"], ms.min(), ms.max(), stats[name]["n_accepted"], stats[name]["n_rejected"],
            stats[name]["nfe"], stats[name]["stage_func"]), flush=True)
    ref = sols["external_eager"]
    res["max_abs_diff_vs_external_eager"] = {k: float((v - ref).abs().max()) for k, v in sols.items()}
    res["linear_fused_equals_unfused"] = bool(torch.equal(sols["linear_eager"], sols["linear_unfused_eager"]))
    res["linear_graph_equals_eager"] = bool(torch.equal(sols["linear_eager"], sols["linear_cuda_graph"]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("linear_bench.py needs a GPU")
    out = dict(gpu=gpu_info(), shape=[M, D], dtype="float64", torch=torch.__version__,
               peaks=dict(hbm_bytes_per_s=PEAK_BW, fp64_tensor_flop_per_s=PEAK_F64, source="H100 SXM data sheet"))
    print(json.dumps(out["gpu"]), flush=True)
    out["kernel"] = kernel_section(a.launches)
    out["solve"] = solve_section(a.runs)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
