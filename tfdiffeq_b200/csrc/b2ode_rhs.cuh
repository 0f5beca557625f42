// b2ode_rhs.cuh -- the library's built-in right-hand sides (tfdiffeq_b200/rhs.py), shared by the persistent fused kernels
// (b2ode_fused.cu) and the stage kernels with a fused right-hand side of the generic path (b2ode.cu).
#pragma once
#include "b2ode_dev.cuh"

// ------------------------------------------------------------------------------------------------
// built-in right-hand sides: explicit mul/add in the order of the torch expressions in rhs.py
// ------------------------------------------------------------------------------------------------
template <typename T>
struct RhsLorenz {   // examples/lorenz_attractor.py:20-37 ; params {sigma, beta, rho}
    static constexpr int D = 3;
    static constexpr int kSmem = 1;      // no staged weights
    static __device__ __forceinline__ void eval(const double *prm, const T * /*sw*/, T /*t*/, const T (&y)[3], T (&dy)[3]) {
        using A = Ar<T>;
        const T sigma = (T)prm[0], beta = (T)prm[1], rho = (T)prm[2];
        dy[0] = A::mul(sigma, A::sub(y[1], y[0]));                          // sigma * (y - x)
        dy[1] = A::sub(A::mul(y[0], A::sub(rho, y[2])), y[1]);              // x * (rho - z) - y
        dy[2] = A::sub(A::mul(y[0], y[1]), A::mul(beta, y[2]));             // x * y - beta * z
    }
};

template <typename T>
struct RhsLotkaVolterra {   // README.md:67-81 ; params {a, b, c, d}
    static constexpr int D = 2;
    static constexpr int kSmem = 1;
    static __device__ __forceinline__ void eval(const double *prm, const T * /*sw*/, T /*t*/, const T (&y)[2], T (&dy)[2]) {
        using A = Ar<T>;
        const T a = (T)prm[0], b = (T)prm[1], c = (T)prm[2], d = (T)prm[3];
        dy[0] = A::sub(A::mul(a, y[0]), A::mul(A::mul(b, y[0]), y[1]));     // a*x - b*x*z
        dy[1] = A::add(A::mul(-c, y[1]), A::mul(A::mul(d, y[0]), y[1]));    // -c*z + d*x*z
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
    static __device__ __forceinline__ void eval(const double *prm, const T *sw, T /*t*/, const T (&y)[2], T (&dy)[2]) {
        using A = Ar<T>;
        const int H = (int)prm[0];
        const bool cube = prm[1] != 0.0;
        const T u0 = cube ? A::mul(A::mul(y[0], y[0]), y[0]) : y[0];
        const T u1 = cube ? A::mul(A::mul(y[1], y[1]), y[1]) : y[1];
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
    static __device__ __forceinline__ float act_dispatch(float a) { return tanhf(a); }
    static __device__ __forceinline__ double act_dispatch(double a) { return tanh(a); }
};


// DETEST class D (tests/DETEST/detest.py:263-283): a two-body orbit, state [x, y, vx, vy] per row; BASELINE config 5 stacks 32
// of them per batch row (dim 128), i.e. the (B, 128) state is (32 B) rows of 4.  r^3 = (x^2 + y^2)^1.5 like the torch module.
template <typename T>
struct RhsKepler {
    static constexpr int D = 4;
    static constexpr int kSmem = 1;
    static __device__ __forceinline__ void eval(const double * /*prm*/, const T * /*sw*/, T /*t*/, const T (&y)[4], T (&dy)[4]) {
        using A = Ar<T>;
        const T r2 = A::add(A::mul(y[0], y[0]), A::mul(y[1], y[1]));
        const T r3 = A::pow(r2, T(1.5));
        dy[0] = y[2];
        dy[1] = y[3];
        dy[2] = A::div(-y[0], r3);
        dy[3] = A::div(-y[1], r3);
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
