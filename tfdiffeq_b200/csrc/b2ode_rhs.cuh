// b2ode_rhs.cuh -- the library's built-in right-hand sides (tfdiffeq_b200/rhs.py), shared by the persistent fused kernels
// (b2ode_fused.cu) and the stage kernels with a fused right-hand side of the generic path (b2ode.cu).
#pragma once
#include "b2ode_dev.cuh"

// ------------------------------------------------------------------------------------------------
// built-in right-hand sides: explicit mul/add in the order of the torch expressions in rhs.py
//
// vjp(prm, sw, t, y, g, f, gy): f = f(t, y) and gy = g^T df/dy for one row, g the row's cotangent (odeint_adjoint passes
// g = -a).  The products and sums are torch autograd's for the module's forward, in the order its engine accumulates them:
// backward nodes run latest-created first, so the contributions to one input element add up in reverse creation order of
// their uses, and the final "+ 0" is the zero-filled select gradient every element is summed with (it turns -0 into +0).
// ------------------------------------------------------------------------------------------------
template <typename T>
struct RhsLorenz {   // examples/lorenz_attractor.py:20-37 ; params {sigma, beta, rho}
    static constexpr int D = 3;
    static constexpr int kSmem = 1;      // no staged weights
    static constexpr bool kParams = false;
    static constexpr bool kAutonomous = true;   // f does not read t
    static __device__ __forceinline__ void eval(const double *prm, const T * /*sw*/, T /*t*/, const T (&y)[3], T (&dy)[3]) {
        using A = Ar<T>;
        const T sigma = (T)prm[0], beta = (T)prm[1], rho = (T)prm[2];
        dy[0] = A::mul(sigma, A::sub(y[1], y[0]));                          // sigma * (y - x)
        dy[1] = A::sub(A::mul(y[0], A::sub(rho, y[2])), y[1]);              // x * (rho - z) - y
        dy[2] = A::sub(A::mul(y[0], y[1]), A::mul(beta, y[2]));             // x * y - beta * z
    }
    static __device__ __forceinline__ void vjp(const double *prm, const T *sw, T t, const T (&y)[3], const T (&g)[3], T (&f)[3],
                                               T (&gy)[3]) {
        using A = Ar<T>;
        eval(prm, sw, t, y, f);
        const T sigma = (T)prm[0], beta = (T)prm[1], rho = (T)prm[2];
        const T g0s = A::mul(g[0], sigma);
        // x: x*y (g2 y), x*(rho - z) (g1 (rho - z)), y - x (-(g0 sigma))
        gy[0] = A::add(A::add(A::add(A::mul(g[2], y[1]), A::mul(g[1], A::sub(rho, y[2]))), -g0s), T(0));
        // y: x*y (g2 x), ... - y (-g1), y - x (g0 sigma)
        gy[1] = A::add(A::add(A::add(A::mul(g[2], y[0]), -g[1]), g0s), T(0));
        // z: beta*z (-g2 beta), rho - z (-(g1 x))
        gy[2] = A::add(A::add(A::mul(-g[2], beta), -A::mul(g[1], y[0])), T(0));
    }
};

template <typename T>
struct RhsLotkaVolterra {   // README.md:67-81 ; params {a, b, c, d}
    static constexpr int D = 2;
    static constexpr int kSmem = 1;
    static constexpr bool kParams = false;
    static constexpr bool kAutonomous = true;
    static __device__ __forceinline__ void eval(const double *prm, const T * /*sw*/, T /*t*/, const T (&y)[2], T (&dy)[2]) {
        using A = Ar<T>;
        const T a = (T)prm[0], b = (T)prm[1], c = (T)prm[2], d = (T)prm[3];
        dy[0] = A::sub(A::mul(a, y[0]), A::mul(A::mul(b, y[0]), y[1]));     // a*x - b*x*z
        dy[1] = A::add(A::mul(-c, y[1]), A::mul(A::mul(d, y[0]), y[1]));    // -c*z + d*x*z
    }
    static __device__ __forceinline__ void vjp(const double *prm, const T *sw, T t, const T (&y)[2], const T (&g)[2], T (&f)[2],
                                               T (&gy)[2]) {
        using A = Ar<T>;
        eval(prm, sw, t, y, f);
        const T a = (T)prm[0], b = (T)prm[1], c = (T)prm[2], d = (T)prm[3];
        // x: (d x) z (g1 z d), (b x) z (-g0 z b), a x (g0 a)
        gy[0] = A::add(A::add(A::add(A::mul(A::mul(g[1], y[1]), d), A::mul(A::mul(-g[0], y[1]), b)), A::mul(g[0], a)), T(0));
        // z: (d x) z (g1 (d x)), -c z (g1 (-c)), (b x) z (-g0 (b x))
        gy[1] = A::add(A::add(A::add(A::mul(g[1], A::mul(d, y[0])), A::mul(g[1], -c)), A::mul(-g[0], A::mul(b, y[0]))), T(0));
    }
};

// examples/ode_demo.py:115-129 (BASELINE config 3): W2 . tanh(W1 . y**3 + b1) + b2, 2 -> H -> 2, H <= 128.
// params {H, cube}; weights staged in shared memory, packed [W1 (2 x H) | b1 (H) | W2 (H x 2) | b2 (2)].
// torch evaluates the two products with cuBLAS (its own FMA order), so this right-hand side agrees with the
// module's forward to rounding, not bit for bit.
template <typename T>
struct RhsCubicMLP {
    static constexpr int D = 2;
    static constexpr int kMaxH = 128;
    static constexpr int kSmem = 2 * kMaxH + kMaxH + 2 * kMaxH + 2;
    static constexpr bool kParams = true;   // 5 H + 2 trainable weights: vjp's parameter sums run in the stage kernel
    static constexpr bool kAutonomous = true;
    static __device__ __forceinline__ T cubed(const bool cube, const T v) { return cube ? Ar<T>::mul(Ar<T>::mul(v, v), v) : v; }
    static __device__ __forceinline__ void eval(const double *prm, const T *sw, T /*t*/, const T (&y)[2], T (&dy)[2]) {
        using A = Ar<T>;
        const int H = (int)prm[0];
        const bool cube = prm[1] != 0.0;
        const T u0 = cubed(cube, y[0]);
        const T u1 = cubed(cube, y[1]);
        const T *W1 = sw, *b1 = sw + 2 * H, *W2 = sw + 3 * H, *b2 = sw + 5 * H;
        T o0 = T(0), o1 = T(0);
        for (int h = 0; h < H; ++h) {
            const T a = A::add(A::add(A::mul(u0, W1[h]), A::mul(u1, W1[H + h])), b1[h]);
            const T z = act_dispatch(a);
            o0 = A::add(o0, A::mul(z, W2[2 * h]));
            o1 = A::add(o1, A::mul(z, W2[2 * h + 1]));
        }
        dy[0] = A::add(o0, b2[0]);
        dy[1] = A::add(o1, b2[1]);
    }
    // hidden unit h of a row with inputs (u0, u1) and cotangent g: z = tanh(u W1 + b1), delta = (W2 g) (1 - z^2)
    static __device__ __forceinline__ void unit(const T *sw, int H, int h, T u0, T u1, const T (&g)[2], T &z, T &delta) {
        using A = Ar<T>;
        const T *W1 = sw, *b1 = sw + 2 * H, *W2 = sw + 3 * H;
        z = act_dispatch(A::add(A::add(A::mul(u0, W1[h]), A::mul(u1, W1[H + h])), b1[h]));
        delta = A::mul(A::add(A::mul(W2[2 * h], g[0]), A::mul(W2[2 * h + 1], g[1])), A::sub(T(1), A::mul(z, z)));
    }
    // f(y) and g^T df/dy = 3 y^2 (W1 delta) (y without the cube); one loop over the hidden units.  The parameter sums
    // (dW1 = u^T delta, db1 = delta, dW2 = z^T g, db2 = g) are taken over all rows by the caller, unit by unit.
    static __device__ __forceinline__ void vjp(const double *prm, const T *sw, T /*t*/, const T (&y)[2], const T (&g)[2],
                                               T (&f)[2], T (&gy)[2]) {
        using A = Ar<T>;
        const int H = (int)prm[0];
        const bool cube = prm[1] != 0.0;
        const T u0 = cubed(cube, y[0]);
        const T u1 = cubed(cube, y[1]);
        const T *W1 = sw, *W2 = sw + 3 * H, *b2 = sw + 5 * H;
        T o0 = T(0), o1 = T(0), s0 = T(0), s1 = T(0);
        for (int h = 0; h < H; ++h) {
            T z, delta;
            unit(sw, H, h, u0, u1, g, z, delta);
            o0 = A::add(o0, A::mul(z, W2[2 * h]));
            o1 = A::add(o1, A::mul(z, W2[2 * h + 1]));
            s0 = A::add(s0, A::mul(W1[h], delta));
            s1 = A::add(s1, A::mul(W1[H + h], delta));
        }
        f[0] = A::add(o0, b2[0]);
        f[1] = A::add(o1, b2[1]);
        gy[0] = cube ? A::mul(s0, A::mul(T(3), A::mul(y[0], y[0]))) : s0;
        gy[1] = cube ? A::mul(s1, A::mul(T(3), A::mul(y[1], y[1]))) : s1;
    }
    static __device__ __forceinline__ float act_dispatch(float a) { return tanhf(a); }
    static __device__ __forceinline__ double act_dispatch(double a) { return tanh(a); }
};


// DETEST class D (tests/DETEST/detest.py:263-283): a two-body orbit, state [x, y, vx, vy] per row; BASELINE config 5 stacks 32
// of them per batch row (dim 128), i.e. the (B, 128) state is (32 B) rows of 4.  r^3 = (x^2 + y^2)^1.5 like the torch module.
template <typename T>
struct RhsKepler {
    static constexpr int D = 4;
    static constexpr int kSmem = 1;
    static constexpr bool kParams = false;
    static constexpr bool kAutonomous = true;
    static __device__ __forceinline__ void eval(const double * /*prm*/, const T * /*sw*/, T /*t*/, const T (&y)[4], T (&dy)[4]) {
        using A = Ar<T>;
        const T r2 = A::add(A::mul(y[0], y[0]), A::mul(y[1], y[1]));
        const T r3 = A::pow(r2, T(1.5));
        dy[0] = y[2];
        dy[1] = y[3];
        dy[2] = A::div(-y[0], r3);
        dy[3] = A::div(-y[1], r3);
    }
    // torch's backward of (x x + y y) ** 1.5 is grad * (1.5 * (x x + y y) ** 0.5), and its CUDA pow special-cases the
    // exponent 0.5 as the correctly rounded sqrt; a / b contributes -grad * ((a / b) / b) to b
    static __device__ __forceinline__ void vjp(const double *prm, const T *sw, T t, const T (&y)[4], const T (&g)[4], T (&f)[4],
                                               T (&gy)[4]) {
        using A = Ar<T>;
        eval(prm, sw, t, y, f);
        const T r2 = A::add(A::mul(y[0], y[0]), A::mul(y[1], y[1]));
        const T r3 = A::pow(r2, T(1.5));
        const T g_r3 = A::add(A::mul(-g[3], A::div(f[3], r3)), A::mul(-g[2], A::div(f[2], r3)));
        const T g_r2 = A::mul(g_r3, A::mul(T(1.5), A::sqrt(r2)));
        // x: -x (-(g2 / r3)), then x * x twice
        gy[0] = A::add(A::add(A::add(-A::div(g[2], r3), A::mul(g_r2, y[0])), A::mul(g_r2, y[0])), T(0));
        gy[1] = A::add(A::add(A::add(-A::div(g[3], r3), A::mul(g_r2, y[1])), A::mul(g_r2, y[1])), T(0));
        gy[2] = A::add(g[0], T(0));
        gy[3] = A::add(g[1], T(0));
    }
};

// ------------------------------------------------------------------------------------------------
// host side: the one place that maps a b2ode_rhs_desc onto the structs above, for every entry point
// ------------------------------------------------------------------------------------------------
static inline int rhs_row_dim(int kind) {
    switch (kind) {
        case B2ODE_RHS_LORENZ: return RhsLorenz<double>::D;
        case B2ODE_RHS_LOTKA_VOLTERRA: return RhsLotkaVolterra<double>::D;
        case B2ODE_RHS_CUBIC_MLP: return RhsCubicMLP<double>::D;
        case B2ODE_RHS_KEPLER: return RhsKepler<double>::D;
    }
    return -1;
}

// Validates `r` for a state of n_elems elements and sets *rows = n_elems / D.  Called before the first CUDA call of every
// entry point, so that a malformed description gets the same code and message whichever entry point it reaches.
static inline int check_rhs(const b2ode_rhs_desc *r, long long n_elems, long long *rows) {
    if (!r) return b2_fail(B2ODE_EINVAL, "null right-hand side");
    const int D = rhs_row_dim(r->kind);
    if (D < 0) return b2_fail(B2ODE_EINVAL, "unknown built-in right-hand side %d", r->kind);
    if (r->n_params < 0 || r->n_params > 8) return b2_fail(B2ODE_EINVAL, "right-hand side n_params %d outside [0, 8]", r->n_params);
    if (n_elems % D != 0) return b2_fail(B2ODE_EINVAL, "state length %lld is not a multiple of the row size %d", n_elems, D);
    if (r->kind == B2ODE_RHS_CUBIC_MLP &&
        (!r->data || r->n_params < 2 || !(r->params[0] >= 1 && r->params[0] <= RhsCubicMLP<double>::kMaxH)))
        return b2_fail(B2ODE_EINVAL, "cubic-MLP right-hand side needs {H in [1, 128], cube} and its weights");
    *rows = n_elems / D;
    return 0;
}

// odeint_adjoint's augmented state for a built-in right-hand side (tfdiffeq/adjoint.py:146): four segments (y, adj_y,
// adj_t, adj_params) of (N, N, 1, max(P, 1)) elements, where P = 5 H + 2 for a B2ODE_RHS_CUBIC_MLP whose weights are all
// trainable and 0 otherwise (adj_params is then the 0-dim zero).  Validates `r` and the layout and sets *rows = N / D and
// *n_params = P.  Called before the first CUDA call of every adjoint entry point, like check_rhs.
static inline int check_adjoint_rhs(const b2ode_rhs_desc *r, int nseg, const int64_t *seg_len, long long *rows, int *n_params) {
    if (nseg != 4 || !seg_len)
        return b2_fail(B2ODE_EINVAL, "the augmented state has 4 segments (y, adj_y, adj_t, adj_params), got %d", nseg);
    const int rc = check_rhs(r, seg_len[0], rows);
    if (rc) return rc;
    if (seg_len[0] < 1 || seg_len[1] != seg_len[0])
        return b2_fail(B2ODE_EINVAL, "adj_y has %lld elements and y %lld: they must be equal and non-zero", (long long)seg_len[1],
                       (long long)seg_len[0]);
    if (seg_len[2] != 1) return b2_fail(B2ODE_EINVAL, "adj_t has %lld elements, not 1", (long long)seg_len[2]);
    int P = 0;
    if (r->kind == B2ODE_RHS_CUBIC_MLP) {
        const int H = (int)r->params[0];
        if (seg_len[3] != 1 && seg_len[3] != 5 * H + 2)
            return b2_fail(B2ODE_EINVAL, "adj_params has %lld elements: a cubic-MLP of hidden width %d takes 1 (frozen weights) or %d",
                           (long long)seg_len[3], H, 5 * H + 2);
        P = seg_len[3] == 1 ? 0 : 5 * H + 2;
    } else if (seg_len[3] != 1) {
        return b2_fail(B2ODE_EINVAL, "adj_params has %lld elements: right-hand side %d has no trainable parameters and takes 1",
                       (long long)seg_len[3], r->kind);
    }
    *n_params = P;
    return 0;
}

// Copies a validated description into a kernel's parameter struct (StageRhsParams, FusedParams and FusedFixedParams name
// the fields alike); parameters past n_params are zero.
template <typename P>
static void fill_rhs(P &p, const b2ode_rhs_desc &r) {
    for (int i = 0; i < 8; ++i) p.rhs[i] = i < r.n_params ? r.params[i] : 0.0;
    p.rhs_data = r.data;
    p.time_sign = r.time_sign;
}

// f(RHS()) with RHS the device struct of `kind` in the state type T: the one switch that picks kernel instantiations.
template <typename T, typename F>
static int dispatch_rhs(int kind, F &&f) {
    switch (kind) {
        case B2ODE_RHS_LORENZ: return f(RhsLorenz<T>());
        case B2ODE_RHS_LOTKA_VOLTERRA: return f(RhsLotkaVolterra<T>());
        case B2ODE_RHS_CUBIC_MLP: return f(RhsCubicMLP<T>());
        case B2ODE_RHS_KEPLER: return f(RhsKepler<T>());
    }
    return b2_fail(B2ODE_EINVAL, "unknown built-in right-hand side %d", kind);
}
