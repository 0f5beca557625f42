"""CPU: the premises of tests/test_exact_gemm_gpu.py -- every case's operands accumulate exactly in fp32, the TF32
emulations agree with their definitions, and the case tables reach the launch geometries they are meant to reach on
an H100 SXM (132 SMs)."""
import numpy as np
import pytest
import torch

import exact_gemm as eg


@pytest.mark.parametrize("case", eg.DENSE_CASES + eg.STAGE_CASES, ids=lambda c: c.name)
def test_dense_case_premise(case):
    ops = eg.dense_operands(case, eg.H100_SMS)
    a = eg.stage_combine(ops["x"], ops["ks"], ops["coefs"])
    bits = eg.premise_bits(eg.dense_terms(a, ops["W"], case.mode), ops["bias"])
    assert float(bits.max()) <= eg.EXACT_BITS, float(bits.max())
    _, pre = eg.dense_expected(ops, case)
    assert np.array_equal(pre.astype(np.float32).astype(np.float64), pre)
    # the stage combine is exact too: A is what the generator meant, whatever the order of the adds
    if case.nk:
        exact = ops["x"].astype(np.float64) + sum(eg.DT * c * k.astype(np.float64) for c, k in zip(ops["coefs"], ops["ks"]))
        assert np.array_equal(a.astype(np.float64), exact)
    if case.mode == "tf32":
        r = eg.tf32_rna(a)
        assert np.count_nonzero(r != eg.tf32_rne(a)) > 0 and np.count_nonzero(r != a) > 0     # RNA ties in A
        assert np.array_equal(eg.tf32_rna(ops["W"]), ops["W"])
    else:
        # both halves of both operands carry bits, and A_lo W_lo (dropped by the kernel) is not zero
        for v in (a, ops["W"]):
            hi, lo = eg.tf32_split(v)
            assert np.mean(lo != 0) > 0.5 and np.all(hi != 0) or case.act in (2, 3)
        assert np.count_nonzero(eg.tf32_split(a)[1][:, 1:] @ eg.tf32_split(ops["W"])[1][:, 1:].T) > 0


@pytest.mark.parametrize("case", eg.MLP3_CASES, ids=lambda c: c.name)
def test_mlp3_case_premise(case):
    ops = eg.mlp3_operands(case, eg.H100_SMS)
    worst, fits = eg.mlp3_premise(ops, case)
    assert worst <= eg.EXACT_BITS and fits, worst
    t1, t2 = eg.hidden_ties(ops, case)
    assert t1 > 0 and t2 > 0, (t1, t2)                          # RNE and RNA differ on some hidden activations
    w1 = ops["W"][0]
    assert np.count_nonzero(eg.tf32_rna(w1) != w1) >= w1.shape[0]        # ties for k_mlp3_pack in every row of W1
    assert np.count_nonzero(eg.tf32_rna(ops["x"]) != ops["x"]) > 0 or case.nk
    # the hidden activations use the bits the Veltkamp constant keeps: rounding to 12 bits would differ
    _, _, pres, _, _ = eg.mlp3_expected(ops, case)
    v = pres[0].astype(np.float32)
    assert np.count_nonzero(eg.tf32_rne(v) != v) > 0


def test_linear_premise():
    for D in eg.LINEAR_DIMS:
        for nk in range(14):
            assert eg.linear_bits(D, nk) <= 50
    lo, hi = eg.linear_blocks_per_warp(eg.linear_rows(eg.H100_SMS), eg.H100_SMS)
    assert lo >= 3 and eg.linear_rows(eg.H100_SMS) % 16


def _all_finite_floats(step):
    """float32 values over every exponent, with mantissa patterns around the TF32 rounding point."""
    e = np.arange(0, 255, dtype=np.uint32) << 23
    mant = np.array([0, 1, 0xFFF, 0x1000, 0x1001, 0x1FFF, 0x2000, 0x3000, 0x5000, 0x7FE000, 0x7FF000, 0x7FFFFF,
                     0x2A5A5A, 0x155000], dtype=np.uint32)
    bits = (e[:, None] | mant[None, :]).ravel()[::step]
    v = bits.view(np.float32)
    return np.concatenate([v, -v])


def test_rna_matches_its_definition_over_all_exponents():
    v = _all_finite_floats(1)
    got = eg.tf32_rna(v)
    want = np.array([eg.tf32_reference(float(x), "away") for x in v], np.float64)
    ok = np.isfinite(want)
    assert np.array_equal(got[ok].astype(np.float64), want[ok])
    # rhs._round_tf32 (the host rounding of W) is the same function
    from tfdiffeq_b200 import rhs
    t = rhs._round_tf32(torch.from_numpy(v.copy())).numpy()
    assert np.array_equal(t.view(np.uint32), got.view(np.uint32))


def test_veltkamp_is_round_to_nearest_even():
    """Over every normal exponent where x * 8193 does not overflow (2^-126 <= |x| < 4e34), and zero.  (On subnormals the
    split keeps 11 significant bits of the value rather than TF32's fixed 2^-136 grid; the kernels never meet them.)"""
    v = _all_finite_floats(1)
    v = v[(np.abs(v) < 4e34) & ((np.abs(v) >= 2.0 ** -126) | (v == 0))]
    got = eg.tf32_rne(v)
    want = np.array([eg.tf32_reference(float(x), "even") for x in v], np.float64)
    assert np.array_equal(got.astype(np.float64), want)


@pytest.mark.parametrize("v,rna,rne", [(1 + 2.0 ** -11, 1 + 2.0 ** -10, 1.0), (2049.0, 2050.0, 2048.0),
                                       (2051.0, 2052.0, 2052.0), (-2049.0, -2050.0, -2048.0),
                                       (2.0 ** -137, 2.0 ** -136, None),                         # fp32 subnormal: RNA only
                                       (1 + 3 * 2.0 ** -12, 1 + 2.0 ** -10, 1 + 2.0 ** -10)])
def test_tie_cases(v, rna, rne):
    x = np.array([v], np.float32)
    assert float(eg.tf32_rna(x)[0]) == rna == eg.tf32_reference(v, "away")
    if rne is not None:
        assert float(eg.tf32_rne(x)[0]) == rne == eg.tf32_reference(v, "even")


def test_case_tables_cover_the_geometry_at_132_sms():
    want_dense = {"ns1", "ns2", "ns3", "ns4", "narrow_last_n_tile", "items3_odd_chunks", "items3_even_chunks",
                  "k_below_chunk", "k_off_chunk", "k_scalar", "partial_m_tile"}
    assert want_dense <= eg.dense_coverage(eg.H100_SMS)
    want_mlp3 = {"stages2", "stages8", "partial_group_layer1", "partial_group_layer3",
                 "ring_uses_not_multiple_of_stages", "tiles3"}
    assert want_mlp3 <= eg.mlp3_coverage(eg.H100_SMS)
    # stage combines for every nk on both producer paths and in both modes
    assert {(c.nk, c.mode, c.K % 4 == 0) for c in eg.STAGE_CASES} == {(nk, m, v) for nk in range(1, 9)
                                                                       for m in ("tf32", "x3") for v in (True, False)}
    assert {c.nk for c in eg.MLP3_CASES} == set(range(9))


def test_geometry_restatement():
    g = eg.dense_geometry(50725, 36, 48, 132, False)
    assert (g.ns, g.tiles_n, g.items, g.grid, g.items_per_cta, g.chunks) == (1, 1, 397, 132, 3, 1)
    g = eg.dense_geometry(25381, 98, 272, 132, True)
    assert (g.ns, g.tiles_n, g.last_nt, g.items, g.chunks) == (4, 2, 16, 398, 6)
    g = eg.mlp3_geometry(4096, 64, 256, 132)
    assert (g.act_bytes, g.stage_bytes, g.stages) == (131072, 32768, 2)
    g = eg.mlp3_geometry(3000, 256, 48, 132)
    assert g.grp == (5, 5, 1) and g.uses == (2, 1, 2)
    assert eg.linear_blocks_per_warp(4099, 132) == (0, 1)
