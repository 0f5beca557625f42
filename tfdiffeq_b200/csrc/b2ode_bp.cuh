// b2ode_bp.cuh -- per-element bodies of the backward pass through the accepted steps, shared by the shared-step kernels
// (k_bp_dense, k_bp_rhs in b2ode.cu) and the independent-rows sweep (k_rows_bp in b2ode_fused.cu), so that both form every
// cotangent with the same operations in the same order.
#pragma once
#include "b2ode_dev.cuh"

// The VJP of one element of the quartic dense output (interp.py:22-36, 55-67): out_j = a x^4 + b x^3 + c x^2 + d x + y0
// with x = (t_out[j] - t0) / den, linear in (y0, y1, f0, f1, y_mid).  gat(j) is the cotangent of output j, j in [j0, j1).
// Returns the cotangents of y0 (a0), y1 (a1), y_mid (gmid) and the dt-scaled ones of f0 and f1.
template <typename T, typename G>
__device__ __forceinline__ void bp_dense_quartic(const G &gat, int j0, int j1, const double *t_out, T t0, T den, T dt, T &a0,
                                                 T &a1, T &gmid, T &f0, T &f1) {
    using A = Ar<T>;
    T GA = T(0), GB = T(0), GC = T(0), GD = T(0), G1 = T(0);
    for (int j = j0; j < j1; ++j) {
        const T gj = gat(j);
        const T x = A::div(A::sub((T)t_out[j], t0), den);
        const T x2 = A::mul(x, x), x3 = A::mul(x2, x), x4 = A::mul(x3, x);
        GA = A::add(GA, A::mul(gj, x4));
        GB = A::add(GB, A::mul(gj, x3));
        GC = A::add(GC, A::mul(gj, x2));
        GD = A::add(GD, A::mul(gj, x));
        G1 = A::add(G1, gj);
    }
    gmid = A::add(A::sub(A::mul(T(16), GA), A::mul(T(32), GB)), A::mul(T(16), GC));
    a0 = A::add(A::sub(A::mul(T(18), GB), A::mul(T(8), GA)), A::mul(T(-11), GC));
    a0 = A::add(A::add(a0, G1), gmid);
    a1 = A::sub(A::sub(A::mul(T(14), GB), A::mul(T(8), GA)), A::mul(T(5), GC));
    f0 = A::add(A::sub(A::mul(T(5), GB), A::mul(T(2), GA)), A::sub(GD, A::mul(T(4), GC)));
    f0 = A::mul(dt, f0);
    f1 = A::mul(dt, A::add(A::sub(A::mul(T(2), GA), A::mul(T(3), GB)), GC));
}

// The dense output's cotangent of k_k (k in the dense output's k mask): (dt c_mid_k) gmid, plus f0's for k = 0 and f1's for
// the last k.
template <typename T>
__device__ __forceinline__ T bp_dense_k(int k, int last, T dt, double c_mid, T gmid, T f0, T f1) {
    T v = Ar<T>::mul(Ar<T>::mul(dt, (T)c_mid), gmid);
    if (k == 0) v = Ar<T>::add(v, f0);
    if (k == last) v = Ar<T>::add(v, f1);
    return v;
}
