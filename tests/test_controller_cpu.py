"""CPU: the step-size controller probes of tests/controller_cases.py -- the restatement against the oracle's controller,
every probe's premises, the engine's controllers emulated on the host within their bounds, and deliberately wrong
controllers outside them."""
import mpmath
import numpy as np
import pytest

import controller_cases as cc
import exact_schedule as es


def _decisions(ps):
    """(probe, attempt index, decision, ratio) of every restated decision of a set."""
    for pr in ps.probes:
        for i, (d, r) in enumerate(zip(pr.decisions, pr.ratios)):
            yield pr, i, d, r


@pytest.mark.parametrize("name", cc.SET_NAMES)
def test_restatement_agrees_with_the_oracle_controller(name):
    """np_ref.optimal_step_size (optimal_step_size_tsit5) on the same state-dtype ratio agrees with the 60-digit
    restatement at every decision of every probe: exactly at m = 0, in the flat band and at the clamps (one correctly
    rounded operation each), else within the oracle's own three roundings (pow, / safety, dt / factor: 3u, plus the
    rounding of the restatement for the comparison)."""
    ps = cc.set_by_name(name)
    for pr, i, d, _ in _decisions(ps):
        got = cc.oracle_dt(pr.dts[i], d.m_T, ps.P, ps.dtype)
        want = float(d.dt_next)
        if d.branch in ("grow", "shrink"):
            assert cc.rel_error(got, d) <= 3 * cc.U, (pr.name, i, d.branch, got, want)
        else:
            assert got == want, (pr.name, i, d.branch, got, want)


@pytest.mark.parametrize("name", cc.SET_NAMES)
def test_probes_meet_their_premises(name):
    ps = cc.set_by_name(name)
    assert [pr.regime for pr in ps.probes] == cc.set_regimes(ps.dtype)
    for pr in ps.probes:
        assert not cc.probe_premises(pr, ps), (pr.name, cc.probe_premises(pr, ps))
        assert pr.dts[0] == ps.h and ps.t[-1] == ps.h / 256
    if ps.method != "tsit5":
        # one trajectory: one block of one trajectory warp in the persistent kernel at 132 SMs
        g = es.fused_geometry(1, cc.H100_SMS, ps.method, ps.dtype, 3)
        assert (g.grid, g.ncw) == (1, 1)
    # the set reaches every branch of the controller
    assert {d.branch for _, _, d, _ in _decisions(ps)} >= {"zero", "ifactor", "grow", "flat", "shrink", "dfactor"}


def test_fp32_window_probes_round_to_one():
    """The window probes' exact ratio lies in [1 - 2^-25, 1): fp32 rounds it to 1.0f (accepted, dfactor kept), fp64
    arithmetic on the unrounded ratio sees m < 1."""
    for name in cc.SET_NAMES:
        ps = cc.set_by_name(name)
        if ps.dtype != "float32":
            continue
        pr = next(p for p in ps.probes if p.regime == "window")
        m = pr.ratios[0].m
        assert cc.mpf(cc.WINDOW[0]) <= m < 1 and np.float32(float(m)) == 1.0
        assert len(pr.decisions) == 1 and pr.decisions[0].branch == "shrink"


@pytest.mark.parametrize("kind", ["last", "zero"])
@pytest.mark.parametrize("dtype", cc.DTYPES)
def test_multi_segment_probes_meet_their_premises(kind, dtype):
    mp = cc.multi_probe(kind, dtype)
    assert not cc.multi_premises(mp), cc.multi_premises(mp)
    assert mp.d.m_T <= 1.0


# --------------------------------------------------------------------------------------------------
# host emulations of ctrl_decide / ctrl_fast
# --------------------------------------------------------------------------------------------------
def _emulated(impl, pr, i, ps, **variant):
    d, r = pr.decisions[i], pr.ratios[i]
    dt = pr.dts[i]
    if impl == "decide":
        with mpmath.workdps(cc.DPS):
            m64 = float(r.m)
        return cc.emulate_decide(dt, m64, ps.P, ps.dtype, **variant)
    return cc.emulate_fast(dt, float(r.ssq[0]), cc.tol2n(ps), ps.P, ps.dtype, **variant)


def _violations(impl, sets, bar, **variant):
    """Decisions of the sets where the emulated controller (with `variant`) misses the restatement by more than its
    bound; bit-exact branches must match exactly."""
    out = []
    for name in sets:
        ps = cc.set_by_name(name)
        for pr, i, d, r in _decisions(ps):
            got = _emulated(impl, pr, i, ps, **variant)
            msg = cc.check_dt(got, d, cc.decision_bound(impl, d, r.ssq[0], ps, bar))
            if msg:
                out.append((name, pr.name, i, msg))
    return out


FAST_SETS = [n for n in cc.SET_NAMES if not n.startswith("tsit5")]


@pytest.mark.parametrize("dtype", cc.DTYPES)
def test_ctrl_decide_emulation_within_bound(dtype):
    sets = [n for n in cc.SET_NAMES if cc.set_by_name(n).dtype == dtype]
    assert not _violations("decide", sets, cc.ratio_bar("stages", dtype, 3))


@pytest.mark.parametrize("dtype", cc.DTYPES)
def test_ctrl_fast_emulation_within_bound(dtype):
    sets = [n for n in FAST_SETS if cc.set_by_name(n).dtype == dtype]
    assert not _violations("fast", sets, cc.ratio_bar("persistent", dtype, 3))


def test_ctrl_fast_old_dfactor_switch_fails_only_in_the_fp32_window():
    """The dfactor switch on the unrounded ratio (ssq < tol^2 n) stays inside the bound everywhere except the fp32
    window, where it keeps dt instead of shrinking it."""
    bad = _violations("fast", FAST_SETS, 1e-12, old_df=True)
    assert bad
    for name, probe, i, _ in bad:
        assert probe == "window" and "-f32-" in name and i == 0, (name, probe)
    assert len(bad) == sum(1 for n in FAST_SETS if "-f32-" in n)


@pytest.mark.parametrize("impl, variant", [
    ("decide", dict(swap_exponent=True)),            # tsit5's exact 1/order swapped with the float32-rounded one
    ("decide", dict(raw_safety=0.9)),                # safety without the float32 rounding of _tf_f64
    ("decide", dict(f32_log2=True)),                 # log2 in fp32 on the chain
    ("fast", dict(f32_log2=True)),
    ("decide", dict(skip_m_round=True)),             # the ratio not rounded to the state dtype
    ("fast", dict(old_df=True)),                     # ctrl_fast's former dfactor switch
])
def test_wrong_controllers_break_a_bound(impl, variant):
    sets = cc.SET_NAMES if impl == "decide" else FAST_SETS
    if "raw_safety" in variant:
        sets = [n for n in sets if n.endswith("-default")]
    bar = cc.ratio_bar("persistent" if impl == "fast" else "stages", "float64", 3)
    assert _violations(impl, sets, bar, **variant)


def test_bounds_are_tight_enough_to_see_an_ulp_level_error():
    """A dt_next off by 1e-9 relative misses every grow / shrink bound of every set."""
    for name in cc.SET_NAMES:
        ps = cc.set_by_name(name)
        for pr, i, d, r in _decisions(ps):
            if d.branch in ("grow", "shrink"):
                for impl, bar in (("decide", cc.ratio_bar("stages", ps.dtype, 3)),
                                  ("fast", cc.ratio_bar("persistent", ps.dtype, 3))):
                    b = cc.decision_bound(impl, d, r.ssq[0], ps, bar)
                    assert b < (1e-9 if ps.dtype == "float64" or impl == "decide" else 1e-7), (name, pr.name, impl, b)
