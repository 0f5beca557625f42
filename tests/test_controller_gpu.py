"""GPU: every kernel family's step-size controller, decision by decision, against the 60-digit restatement of
tests/controller_cases.py, under the default options and safety=0.8, ifactor=5, dfactor=0.3.

Every probe of a (tableau, dtype, options) set runs through each controller site: the persistent kernel (ctrl_fast), the
stage kernels, the generic path with a torch func (eager, and with cuda_graph, which replays every attempt after the
first), and all probes of the set as the rows of one independent_rows launch (all ctrl_decide).  tsit5 runs on the
generic path only.  Per probe: the accepted and rejected counts, the reported ratio of the last attempt, and dt_next
within the implementation's bound -- bit for bit in the flat band, and dt * ifactor exactly at m = 0.  Where two
ctrl_decide sites report the same ratio bits for a one-attempt probe, their dt_next bits are equal.
tests/test_controller_cpu.py checks the probes' premises."""
import mpmath
import numpy as np
import pytest
import torch

import controller_cases as cc
from problems import PROBLEMS

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
DECIDE_SITES = ("stages", "func", "func_graph", "rows")
WORST = {}       # family -> (largest error in u, its bound in u, where)


def tfd():
    import tfdiffeq_b200
    return tfdiffeq_b200


def _options(ps, **extra):
    return dict(cc.OPTION_SETS[ps.opts], first_step=ps.h, **extra)


def _run(site, func, y0, ps):
    """(n_acc, n_rej, dt_next, ratio) of a one-trajectory solve at a site.  With cuda_graph the first attempt runs eagerly
    and the later ones replay a graph, so the graph carries the later decisions of rejecting probes."""
    y = torch.tensor(y0, device=DEV)
    extra = {"persistent": {}, "stages": dict(fused_rhs="stages"), "func": {}, "func_graph": dict(cuda_graph=True)}[site]
    tfd().odeint(func, y, torch.tensor(ps.t), rtol=0.0, atol=ps.atol, method=ps.method, options=_options(ps, **extra))
    st = dict(tfd().last_stats)
    if site == "persistent":
        assert st["fused_rhs"] and not st["stage_rhs"], st
    elif site == "stages":
        assert st["stage_rhs"] and not st["fused_rhs"], st
    else:
        graph = site == "func_graph" and st["n_rejected"] > 0
        assert not st["stage_rhs"] and not st["fused_rhs"] and st["cuda_graph"] == graph, st
    return st["n_accepted"], st["n_rejected"], st["dt_next"], st["error_ratio"]


def _rows(ps):
    """Every probe of the set as one row of a single independent_rows launch."""
    y0 = np.concatenate([pr.y0 for pr in ps.probes])
    tfd().odeint(tfd().rhs.Lorenz(), torch.tensor(y0, device=DEV), torch.tensor(ps.t), rtol=0.0, atol=ps.atol,
                 method=ps.method, options=_options(ps, independent_rows=True))
    st = tfd().last_stats
    assert st["independent_rows"] and st["rows"] == len(ps.probes)
    cols = [st[k].cpu().numpy() for k in ("row_accepted", "row_rejected", "row_dt_next", "row_error_ratio")]
    return [(int(a), int(r), float(d), float(m)) for a, r, d, m in zip(*cols)]


def _check(site, pr, ps, got):
    """Failures of one probe at one site (an empty list when it passes)."""
    n_acc, n_rej, dt_next, ratio = got
    impl = "fast" if site == "persistent" else "decide"
    family = "persistent" if site == "persistent" else "ctrl_decide"
    bar = cc.ratio_bar(family, ps.dtype, 3)
    k = len(pr.decisions)
    bad = []
    if (n_acc, n_rej) != (1, k - 1):
        bad.append("counts %d/%d, want 1/%d" % (n_acc, n_rej, k - 1))
        return bad
    m_last = pr.ratios[-1].m
    tol = cc.ratio_tolerance(pr, ps, bar, impl)
    if tol == 0.0:
        if ratio != cc.round_to(m_last, ps.dtype):
            bad.append("ratio %r != %r" % (ratio, cc.round_to(m_last, ps.dtype)))
    else:
        with mpmath.workdps(cc.DPS):
            rel = float(abs(cc.mpf(ratio) / m_last - 1)) if m_last != 0 else abs(ratio)
        if rel > tol:
            bad.append("ratio %r: rel. error %.3e > %.3e" % (ratio, rel, tol))
    if k == 1:
        d = pr.decisions[0]
        bound = cc.decision_bound(impl, d, pr.ratios[0].ssq[0], ps, bar)
    else:
        # the last decision restated at the reported ratio, from the restated step of the last attempt
        d = cc.final_decision(pr, ps, ratio)
        if d.branch != pr.decisions[-1].branch:
            bad.append("last decision %s, want %s" % (d.branch, pr.decisions[-1].branch))
        ssq = ratio * cc.tol2n(ps)
        bound = cc.chain_bound(impl, pr, ps, bar) + cc.decision_bound(impl, d, ssq, ps, 4 * cc.U)
    msg = cc.check_dt(dt_next, d, bound)
    if msg:
        bad.append("dt_next %r: %s" % (dt_next, msg))
    if pr.regime == "zero" and dt_next != ps.h * ps.P.ifactor:
        bad.append("m = 0: dt_next %r != dt * ifactor %r" % (dt_next, ps.h * ps.P.ifactor))
    if bound > 0:
        key = "%s %s" % (family, ps.dtype)
        err = cc.rel_error(dt_next, d) / cc.U
        if err / (bound / cc.U) > WORST.get(key, (0, 1, ""))[0] / WORST.get(key, (0, 1, ""))[1]:
            WORST[key] = (err, bound / cc.U, "%s %s %s" % (ps.name, pr.name, site))
    return bad


@pytest.mark.parametrize("name", cc.SET_NAMES)
def test_controller_decisions(name):
    ps = cc.set_by_name(name)
    tsit5 = ps.method == "tsit5"
    sites = ("stages", "func", "func_graph") if tsit5 else ("persistent",) + DECIDE_SITES
    results = {}
    builtin, torch_func = tfd().rhs.Lorenz(), PROBLEMS["lorenz"](backend="torch", device=DEV)
    for site in sites:
        if site == "rows":
            for pr, got in zip(ps.probes, _rows(ps)):
                results[pr.name, site] = got
            continue
        for pr in ps.probes:
            func = builtin if site in ("persistent", "stages") else torch_func
            results[pr.name, site] = _run(site, func, pr.y0, ps)
    failures = []
    for (probe, site), got in results.items():
        pr = next(p for p in ps.probes if p.name == probe)
        failures += ["%s @ %s: %s" % (probe, site, b) for b in _check(site, pr, ps, got)]
    # ctrl_decide is one function: the same ratio bits give the same dt_next bits at every site
    for pr in ps.probes:
        if len(pr.decisions) == 1:
            seen = {}
            for site in sites:
                if site in DECIDE_SITES:
                    _, _, dt_next, ratio = results[pr.name, site]
                    if ratio in seen and seen[ratio][1] != dt_next:
                        failures.append("%s: %s and %s report ratio %r but dt_next %r and %r" % (
                            pr.name, seen[ratio][0], site, ratio, seen[ratio][1], dt_next))
                    seen.setdefault(ratio, (site, dt_next))
    for key, (err, bound, where) in sorted(WORST.items()):
        print("largest dt_next error, %s: %.2f u (bound %.2f u) at %s" % (key, err, bound, where))
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("kind", ["last", "zero"])
@pytest.mark.parametrize("dtype", cc.DTYPES)
def test_multi_segment_controller(kind, dtype):
    """A tuple of three Lorenz batches with per-component tolerances on the generic path: the largest ratio is the last
    component's, or one component sits at the origin with m = 0."""
    mp = cc.multi_probe(kind, dtype)
    f = PROBLEMS["lorenz"](backend="torch", device=DEV)
    y = tuple(torch.tensor(a, device=DEV) for a in mp.y0)
    opts = dict(cc.OPTION_SETS["default"], first_step=mp.h)
    tfd().odeint(lambda t, z: tuple(f(t, c) for c in z), y, torch.tensor(mp.t), rtol=mp.rtol, atol=mp.atol,
                 method="dopri5", options=opts)
    st = tfd().last_stats
    assert (st["n_accepted"], st["n_rejected"]) == (1, 0) and not st["fused_rhs"] and not st["stage_rhs"]
    m = mp.ratio.ms[mp.argmax]
    if dtype == "float32":
        assert st["error_ratio"] == cc.round_to(m, dtype)
    else:
        with mpmath.workdps(cc.DPS):
            assert float(abs(cc.mpf(st["error_ratio"]) / m - 1)) <= cc.ratio_bar("ctrl_decide", dtype, mp.ratio.n[mp.argmax])
    bar = cc.ratio_bar("ctrl_decide", dtype, max(mp.ratio.n))
    bound = cc.dt_bound("decide", mp.d, mp.P, dtype, bar)
    assert cc.check_dt(st["dt_next"], mp.d, bound) is None, cc.check_dt(st["dt_next"], mp.d, bound)
