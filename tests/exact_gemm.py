"""Exact operands for the TF32 tensor-core kernels (b2ode_mma.cu): k_dense_layer_tf32 (single pass and 3xTF32),
k_mlp3_tf32 with k_mlp3_pack, and the fp64 k_linear_f64.

If every product that reaches an fp32 accumulator, the bias and every partial sum are multiples of 2^-q, and
sum |terms| + |bias| <= 2^(22 - q), every addition is exact in fp32 -- in any order, and whether the hardware rounds or
truncates when it aligns the terms, as long as it keeps the 24 significant bits an fp32 result needs (the bound leaves
two bits of margin).  On such operands the kernel has exactly one correct output, and an fp64 (or int64) product of the
operands the tensor core sees -- exact in any summation order -- is a valid reference for ``torch.equal``.  The grid and
the bound are per output element, so rows may carry different power-of-two scales.

What the tensor core sees, restated here:
  * single-pass TF32: A = cvt.rna(x) (ties away from zero), W rounded by the host (``rhs._round_tf32``) or, for the
    chained kernel, by k_mlp3_pack (cvt.rna as well);
  * 3xTF32: A_lo.W_hi + A_hi.W_lo + A_hi.W_hi with hi = rna(v), lo = rna(v - hi) -- A_lo.W_lo is dropped, so the exact
    answer is the three cross products, not the full product;
  * chained kernel: hidden activations rounded by Veltkamp's split (x * 8193, three fp32 operations: round to nearest,
    ties to even), emulated here in numpy float32.

This module is a plain helper (no fixtures): tests/test_exact_gemm_cpu.py checks every premise on the host, and
tests/test_exact_gemm_gpu.py runs the kernels on the same operands.
"""
import collections
from fractions import Fraction
import math

import numpy as np

H100_SMS = 132                 # SMs of an H100 SXM: the geometry the CPU test checks

# b2ode_mma.cu constants
TILE_M, KCHUNK, NSUB, KSUB = 128, 64, 64, 32
MAX_RING, RING_TAIL, BULK_SMEM = 8, 8192, 227 * 1024 - 4096
LIN_WARPS = 8
EXACT_BITS = 22                # sum |terms| <= 2^(22 - q): two bits below fp32's 24


# --------------------------------------------------------------------------------------------------
# TF32 rounding
# --------------------------------------------------------------------------------------------------
def tf32_rna(x):
    """cvt.rna.tf32.f32 on float32 values: keep 10 explicit mantissa bits, round to nearest, ties away from zero."""
    i = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((i + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)


def tf32_rne(x):
    """The chained kernel's to_tf32_fast: Veltkamp's split with C = 2^13 + 1, three IEEE float32 operations."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        g = x * np.float32(8193.0)
        d = x - g
        return g + d


def tf32_split(x):
    """(hi, lo) of the 3xTF32 split: hi = rna(x), lo = rna(x - hi) (the subtraction is exact in fp32)."""
    x = np.asarray(x, dtype=np.float32)
    hi = tf32_rna(x)
    return hi, tf32_rna(x - hi)


def tf32_reference(v, ties):
    """TF32 rounding of one finite float32 value from its definition in exact arithmetic: 11 significant bits (fp32
    subnormals: the same 13 low encoding bits dropped), ties 'away' or 'even'."""
    v = Fraction(float(v))
    if v == 0:
        return 0.0
    _, e = math.frexp(abs(float(v)))                  # |v| = f 2^e, 0.5 <= f < 1
    ulp = Fraction(2) ** max(e - 11, -136)
    n, r = divmod(abs(v), ulp)
    half = Fraction(1, 2)
    up = r / ulp > half or (r / ulp == half and (ties == "away" or n % 2 == 1))
    out = (n + (1 if up else 0)) * ulp
    if out >= 2 ** 128:                               # rounded past FLT_MAX
        out = math.inf
    return float(out if v > 0 else -out)


# --------------------------------------------------------------------------------------------------
# launch geometry, restated from the host code of b2ode_mma.cu
# --------------------------------------------------------------------------------------------------
DenseGeometry = collections.namedtuple("DenseGeometry", "ns tiles_m tiles_n items grid items_per_cta last_nt kchunks chunks")


def dense_geometry(M, K, N, sms, x3):
    """launch_dense / k_dense_layer_tf32: N tile 64 NS wide, items = M tiles x N tiles, one CTA per SM at most;
    an item runs kchunks K chunks per pass (three passes in 3xTF32)."""
    ns = 4 if N >= 256 else -(-N // NSUB)
    ntile = ns * NSUB
    tiles_m, tiles_n = -(-M // TILE_M), -(-N // ntile)
    items = tiles_m * tiles_n
    grid = min(items, sms)
    kchunks = -(-K // KCHUNK)
    return DenseGeometry(ns, tiles_m, tiles_n, items, grid, items // grid, N - (tiles_n - 1) * ntile, kchunks,
                         3 * kchunks if x3 else kchunks)


Mlp3Geometry = collections.namedtuple("Mlp3Geometry", "act_bytes stage_bytes stages grp subs uses ring_uses tiles grid tiles_per_cta")


def mlp3_geometry(M, D, H, sms):
    """b2ode_mlp3 / k_mlp3_tf32: ACT tile, weight ring of `stages` stages of max(D, H) x 128 bytes, K blocks per stage
    (grp) and stage uses (ring acquisitions) per layer, one tile of 128 rows per CTA iteration."""
    blocks_in, blocks_h = 2 * -(-D // KCHUNK), -(-H // KSUB)
    act_bytes = max(blocks_in, blocks_h) * TILE_M * 128
    stage_bytes = max(H, D) * 128
    stages = min((BULK_SMEM - 1024 - act_bytes - RING_TAIL) // stage_bytes, MAX_RING)
    nl = (H, H, D)
    subs = (-(-D // KSUB), -(-H // KSUB), -(-H // KSUB))
    grp = tuple(stage_bytes // (n * 128) for n in nl)
    uses = tuple(-(-s // g) for s, g in zip(subs, grp))
    tiles = -(-M // TILE_M)
    grid = min(tiles, sms)
    return Mlp3Geometry(act_bytes, stage_bytes, stages, grp, subs, uses, sum(uses), tiles, grid, tiles // grid)


def linear_blocks_per_warp(M, sms):
    """launch_linear / k_linear_f64: (fewest, most) 16-row blocks a warp walks (block b, b + 8 grid, ...)."""
    blocks = -(-M // 16)
    grid = min(-(-blocks // LIN_WARPS), sms)
    warps = grid * LIN_WARPS
    return blocks // warps, -(-blocks // warps)


# --------------------------------------------------------------------------------------------------
# operands
# --------------------------------------------------------------------------------------------------
DT = 0.125                                     # dyadic step; dt * coef is exact in fp32
COEFS = [8.0, -16.0, 24.0, 4.0, -8.0, 16.0, -24.0, 40.0, -4.0, 8.0, -16.0, 24.0, -40.0]   # dt * coef in {+-0.5 .. +-5}


def _stage_split(rng, A, nk, scale):
    """(x, ks, coefs) with x + sum_j (dt coef_j) k_j == A exactly in fp32 (k_j even integers times the row scale)."""
    coefs = COEFS[:nk]
    ks = [(2 * rng.integers(-20, 21, size=A.shape)).astype(np.float64) * scale for _ in range(nk)]
    s = np.zeros(A.shape)
    for c, k in zip(coefs, ks):
        s = s + (DT * c) * k
    return (A - s).astype(np.float32), [k.astype(np.float32) for k in ks], coefs


def stage_combine(x, ks, coefs, dt=DT):
    """k_rk_stage's order in float32: c_j = fl(fl(dt) fl(coef_j)), acc = c_0 k_0, acc += c_j k_j, y = x + acc."""
    if not ks:
        return np.asarray(x, np.float32)
    c = [np.float32(dt) * np.float32(b) for b in coefs]
    acc = c[0] * ks[0]
    for cj, kj in zip(c[1:], ks[1:]):
        acc = acc + cj * kj
    return (x + acc).astype(np.float32)


def _split_values(rng, shape, hs):
    """h + j 2^-12 with h in +-hs, j in -3..3, restricted to the pairs whose TF32 split is exactly (h, j 2^-12)."""
    pairs = []
    for h in hs:
        for s in (1, -1):
            for j in range(-3, 4):
                v = np.float32(s * h + j * 2.0 ** -12)
                hi, lo = tf32_split(np.array([v]))
                if hi[0] == s * h and lo[0] == np.float32(j * 2.0 ** -12):
                    pairs.append(float(v))
    return rng.choice(np.array(pairs), size=shape)


DenseCase = collections.namedtuple("DenseCase", "name M K N nk mode act bias")


def _rows_for_items(per_cta, tiles_n, partial=37):
    """M with at least `per_cta` items per CTA at 132 SMs (and any other count), plus a partial last M tile."""
    return lambda sms: TILE_M * (per_cta * sms // tiles_n) + partial


SPECIAL_ACT = [20.0, 20.5, 21.0, 19.75, 40.0, -89.0, -100.0, -150.0, 9.5, -9.5, 12.0, 0.0, -0.5, 0.25]


def dense_operands(case, sms, seed=0):
    """x [M, K], ks, coefs, W [N, K] (fp32, W as given to the host rounding), bias [N] or None, and row scales.

    tf32: the A the tensor core sees is an integer of up to 12 bits (odd values in 2048..4095 are RNA ties) times a
    row scale; W small integers.  x3: every A and W entry is h + j 2^-12 with both halves non-zero.  act 2 / 3 rows are
    scaled into tanh's / softplus's interesting range, and the last rows hold single special arguments through a unit
    first column of W."""
    M = case.M(sms) if callable(case.M) else case.M
    K, N = case.K, case.N
    rng = np.random.default_rng([seed, M, K, N, case.nk, case.act, 1 if case.mode == "x3" else 0])
    if case.mode == "tf32":
        A = rng.integers(-4095, 4096, size=(M, K)).astype(np.float64)
        wmax = max(1, int(2 ** 20 // (K * 2048)))
        W = rng.integers(-wmax, wmax + 1, size=(N, K)).astype(np.float64)
        grid = 1.0
    else:
        A = _split_values(rng, (M, K), (1, 2, 3))
        W = _split_values(rng, (N, K), (1, 2) if K > 100 else (1, 2, 3))
        grid = 2.0 ** -12
    if case.act in (2, 3):
        # bring the pre-activations to O(1 .. 30), where tanh and softplus are not trivial
        e = np.ceil(np.log2(np.median((np.abs(A) @ np.abs(W).T).max(axis=1)))) - 5
        scale = np.full((M, 1), 2.0 ** -e)
    else:
        scale = np.exp2(rng.integers(-3, 4, size=M))[:, None]
    A = A * scale
    bias = None
    if case.bias:
        # on the coarsest row grid (a multiple of every row's grid), small next to the bound
        b_grid = grid * float(scale.max())
        bias = rng.integers(-64, 65, size=N).astype(np.float64) * b_grid
    if case.act in (2, 3):
        W[0, :] = 0.0
        W[:, 0] = 0.0
        W[0, 0] = 1.0
        if bias is not None:
            bias[0] = 0.0
        n = min(len(SPECIAL_ACT), M // 2)
        A[M - n:, :] = 0.0
        A[M - n:, 0] = SPECIAL_ACT[:n]
    x, ks, coefs = _stage_split(rng, A, case.nk, scale) if case.nk else (A.astype(np.float32), [], [])
    return dict(x=x, ks=ks, coefs=coefs, W=W.astype(np.float32), bias=None if bias is None else bias.astype(np.float32))


def dense_terms(a, W, mode):
    """The products the tensor core accumulates, as fp64 matrices whose sum is the exact pre-bias result:
    [rna(a) rna(W)^T] (tf32) or [a_lo W_hi^T, a_hi W_lo^T, a_hi W_hi^T] (x3).  a is the stage input (float32)."""
    if mode == "tf32":
        return [(tf32_rna(a).astype(np.float64), tf32_rna(W).astype(np.float64))]
    ah, al = tf32_split(a)
    wh, wl = tf32_split(W)
    d = np.float64
    return [(al.astype(d), wh.astype(d)), (ah.astype(d), wl.astype(d)), (ah.astype(d), wh.astype(d))]


def _grid_exponent(v):
    """Per element: t with v = n 2^t, n odd (the grid v lies on); +inf for 0."""
    v = np.abs(np.asarray(v, np.float64))
    out = np.full(v.shape, np.inf)
    nz = v != 0
    m, e = np.frexp(v[nz])
    mant = (m * 2.0 ** 53).astype(np.int64)
    out[nz] = e - 53 + np.log2((mant & -mant).astype(np.float64))
    return out


def premise_bits(pairs, bias):
    """Per output element: log2(sum |terms| + |bias|) - (exponent of the finest grid any term or the bias lies on).
    Exact accumulation needs this <= 22 everywhere.  The grid of a term a_k w_k is grid(a_k) + grid(w_k)."""
    total = None
    q = None
    for a, w in pairs:
        s = np.abs(a) @ np.abs(w).T
        total = s if total is None else total + s
        ga, gw = _grid_exponent(a).astype(np.float32), _grid_exponent(w).astype(np.float32)
        if q is None:
            q = np.full(s.shape, np.inf, np.float32)
        for k in range(a.shape[1]):
            np.minimum(q, ga[:, k, None] + gw[None, :, k], out=q)
    if bias is not None:
        total = total + np.abs(bias.astype(np.float64))[None, :]
        q = np.minimum(q, _grid_exponent(bias.astype(np.float64))[None, :])
    with np.errstate(divide="ignore"):
        return np.log2(np.maximum(total, 1e-300)) - q


def dense_expected(ops, case):
    """Exact output (fp64) of the dense layer for the pre-activation terms, act 0 / 1; plus the exact pre-activation."""
    a = stage_combine(ops["x"], ops["ks"], ops["coefs"])
    pre = sum(aa @ ww.T for aa, ww in dense_terms(a, ops["W"], case.mode))
    if ops["bias"] is not None:
        pre = pre + ops["bias"].astype(np.float64)[None, :]
    return a, pre


# the dense-layer case table: NS 1..4, two N tiles with a narrower last one, several items per CTA with odd and even
# chunk counts per item, K below one chunk, K off the chunk and K % 4 != 0 (the element-wise producer)
DENSE_CASES = [
    DenseCase("ns1_k36_items3", _rows_for_items(3, 1), 36, 48, 0, "tf32", 1, True),
    DenseCase("ns2_k100_items3", _rows_for_items(3, 1), 100, 128, 0, "tf32", 0, True),
    DenseCase("ns3_k130", 1000, 130, 176, 0, "tf32", 1, False),
    DenseCase("ns4_2tiles_k7", _rows_for_items(3, 2), 7, 320, 0, "tf32", 0, True),
    DenseCase("ns4_k64", 300, 64, 256, 0, "tf32", 1, True),
    DenseCase("x3_ns1_k36_items3", _rows_for_items(3, 1), 36, 48, 0, "x3", 1, True),
    DenseCase("x3_ns2_k100", 1000, 100, 128, 0, "x3", 0, False),
    DenseCase("x3_ns3_k130", 500, 130, 144, 0, "x3", 0, True),
    DenseCase("x3_ns4_2tiles_k98", _rows_for_items(3, 2), 98, 272, 0, "x3", 1, True),
    DenseCase("tanh_k100", 700, 100, 64, 0, "tf32", 2, True),
    DenseCase("softplus_k36", 700, 36, 64, 0, "tf32", 3, True),
    DenseCase("x3_tanh_k98", 700, 98, 64, 0, "x3", 2, False),
    DenseCase("x3_softplus_k64", 700, 64, 64, 0, "x3", 3, True),
]
# the stage-combine producer for every nk: vector (K = 100) and element-wise (K = 98) paths, both modes
STAGE_CASES = [DenseCase("nk%d_%s_%s" % (nk, mode, path), 1000 + 37 * nk, 100 if path == "vec" else 98, 64, nk, mode, 1, True)
               for nk in range(1, 9) for mode in ("tf32", "x3") for path in ("vec", "scalar")]


# --------------------------------------------------------------------------------------------------
# the chained kernel
# --------------------------------------------------------------------------------------------------
Mlp3Case = collections.namedtuple("Mlp3Case", "name M D H act nk")

MLP3_CASES = [
    Mlp3Case("s2_d256_h256", 4096 + 37, 256, 256, 1, 0),                              # two ring stages
    Mlp3Case("s8_d16_h16_tiles3", lambda sms: TILE_M * 3 * sms + 5, 16, 16, 1, 0),    # eight stages, 3 tiles per CTA
    Mlp3Case("grp1_partial_d256_h48", 3000, 256, 48, 1, 0),                           # D > H: 5 K blocks per stage, 8 in layer 1
    Mlp3Case("grp3_partial_d48_h208", lambda sms: TILE_M * 3 * sms + 77, 48, 208, 0, 0),   # D < H: layer 3 groups 4, 7 blocks
    Mlp3Case("d64_h128_none", 5000, 64, 128, 0, 0),
    Mlp3Case("d112_h80", 777, 112, 80, 1, 0),
] + [Mlp3Case("nk%d_d64_h96" % nk, 1500 + 11 * nk, 64, 96, 1, nk) for nk in range(1, 9)]


def mlp3_operands(case, sms, seed=0):
    """Input whose TF32 rounding is an integer of up to 12 bits (many RNA ties); weights sparse small integers (6, 4 and
    4 non-zeros per row in the three layers, so every layer keeps its pre-activations around 2^12 .. 2^14, where TF32 rounding of the
    hidden activations moves bits and hits ties) plus RNA ties for k_mlp3_pack: +-(1 + 2^-11) 2^p in the first K
    column, where the input is 0 or +-2^10 / +-2^11 so that every product stays an integer."""
    M = case.M(sms) if callable(case.M) else case.M
    D, H = case.D, case.H
    rng = np.random.default_rng([seed, M, D, H, case.act, case.nk])
    A = rng.integers(-4095, 4096, size=(M, D)).astype(np.float64)
    A[:, 0] = rng.choice([0.0, 1024.0, -1024.0, 2048.0, -2048.0], size=M)

    def weight(n, k, tie, nnz, vals):
        w = np.where(rng.random((n, k)) < min(1.0, nnz / k), rng.choice(np.array(vals), size=(n, k)), 0.0)
        if tie:
            w[:, 0] = rng.choice([1.0, -1.0], size=n) * (1.0 + 2.0 ** -11) * np.exp2(rng.integers(0, 2, size=n))
        return w.astype(np.float32)
    W1 = weight(H, D, True, 6, [1.0, -1.0, 2.0, -2.0, 3.0, -3.0, 5.0, -7.0])
    W2 = weight(H, H, False, 4, [1.0, -1.0, 2.0, -3.0])
    W3 = weight(D, H, False, 4, [1.0, -1.0, 3.0, -2.0])
    b1 = rng.integers(-512, 513, size=H).astype(np.float32)
    b2 = rng.integers(-512, 513, size=H).astype(np.float32)
    b3 = rng.integers(-512, 513, size=D).astype(np.float32)
    ones = np.ones((M, 1))
    x, ks, coefs = _stage_split(rng, A, case.nk, ones) if case.nk else (A.astype(np.float32), [], [])
    return dict(x=x, ks=ks, coefs=coefs, W=(W1, W2, W3), b=(b1, b2, b3))


def mlp3_expected(ops, case):
    """Exact chain on the host: layer pre-activations in fp64 (exact under the premise), hidden activations relu'd (or
    not) and rounded by the Veltkamp emulation.  Returns (stage input, output, [pre1, pre2, pre3], [A, h1, h2], W's)."""
    a = stage_combine(ops["x"], ops["ks"], ops["coefs"])
    Ws = [tf32_rna(w).astype(np.float64) for w in ops["W"]]
    h = tf32_rna(a).astype(np.float64)
    ins, pres = [h], []
    for layer in range(3):
        p = h @ Ws[layer].T + ops["b"][layer].astype(np.float64)[None, :]
        pres.append(p)
        if layer < 2:
            v = np.maximum(p, 0.0) if case.act == 1 else p
            h = tf32_rne(v.astype(np.float32)).astype(np.float64)
            ins.append(h)
    return a, pres[2], pres, ins, Ws


def mlp3_premise(ops, case):
    """Worst premise_bits over the three layers, and whether each pre-activation is exactly an fp32 value."""
    _, _, pres, ins, Ws = mlp3_expected(ops, case)
    worst = max(float(premise_bits([(h, w)], b).max()) for h, w, b in zip(ins, Ws, ops["b"]))
    fits = all(np.array_equal(p.astype(np.float32).astype(np.float64), p) for p in pres)
    return worst, fits


def hidden_ties(ops, case):
    """Hidden pre-activations (after the activation) on an RNE/RNA tie where the two differ, per layer."""
    _, _, pres, _, _ = mlp3_expected(ops, case)
    out = []
    for p in pres[:2]:
        v = (np.maximum(p, 0.0) if case.act == 1 else p).astype(np.float32)
        out.append(int(np.count_nonzero(tf32_rne(v) != tf32_rna(v))))
    return out


# --------------------------------------------------------------------------------------------------
# the fp64 linear kernel
# --------------------------------------------------------------------------------------------------
LINEAR_DIMS = (16, 48, 128)


def linear_rows(sms):
    """At least three 16-row blocks for every warp of the persistent grid, and M % 16 != 0."""
    return 3 * 16 * LIN_WARPS * sms + 5


def dense_coverage(sms):
    """Launch features the dense-layer case tables reach on a device of `sms` SMs."""
    seen = set()
    for c in DENSE_CASES + STAGE_CASES:
        M = c.M(sms) if callable(c.M) else c.M
        g = dense_geometry(M, c.K, c.N, sms, c.mode == "x3")
        seen.add("ns%d" % g.ns)
        if g.tiles_n >= 2 and g.last_nt < g.ns * NSUB:
            seen.add("narrow_last_n_tile")
        if g.items_per_cta >= 3:
            seen.add("items3_%s_chunks" % ("odd" if g.chunks % 2 else "even"))
        if c.K < KCHUNK:
            seen.add("k_below_chunk")
        if c.K % KCHUNK:
            seen.add("k_off_chunk")
        if c.K % 4:
            seen.add("k_scalar")
        if M % TILE_M:
            seen.add("partial_m_tile")
    return seen


def mlp3_coverage(sms):
    seen = set()
    for c in MLP3_CASES:
        M = c.M(sms) if callable(c.M) else c.M
        g = mlp3_geometry(M, c.D, c.H, sms)
        seen.add("stages%d" % g.stages)
        for layer in (0, 2):
            if g.grp[layer] > 1 and g.subs[layer] % g.grp[layer]:
                seen.add("partial_group_layer%d" % (layer + 1))
        if g.ring_uses % g.stages:
            seen.add("ring_uses_not_multiple_of_stages")
        if g.tiles_per_cta >= 3:
            seen.add("tiles3")
    return seen


def linear_bits(D, nk):
    """Worst-case bits of the fp64 products on the operands of tests/test_exact_gemm_gpu.py: Y = x + sum_j c_j k_j with
    |x| <= 2^10, |k_j| <= 40 (even), |c_j| <= 5 on the grid 2^-0 .. (integers: dt coef_j k_j is an integer), A integers
    |A| <= 2^10: sum |terms| <= D (2^10 + 5 * 40 nk) 2^10, against fp64's 53 bits."""
    return math.log2(D * (2 ** 10 + 5 * 40 * nk) * 2 ** 10)
