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
//
// Parameter hooks (kParams): the kernels that sum g^T df/dtheta over rows (k_rk_stage_adjoint_rhs, k_bp_rhs, k_rows_bp
// through par_tiles / par_block_partial below) stage tiles of rows in shared memory and call
//   n_weights(prm)             P, the weights staged in sw and the length of the flattened parameter vector
//   tile_rows(NT), kTileVals   rows a tile holds (a divisor of the block's NT threads), values staged per row (at most;
//                              with tiles smaller than the block, tile_vals(prm) is the count)
//   acc_count(NT)              fp64 accumulators per thread
//   stage(prm, sw, y, g, t, ld)            one row's tile values, t[v * ld], from its stage input y and cotangent g
//   accumulate<NT>(prm, sw, tile, on, acc) adds, in row order, the tile rows whose on[] is set to the thread's sums
//   partial<NT>(prm, red, pp)             the block's sums (thread x's accumulator q at red[q * NT + x]) combined in a
//                                          fixed order into pp[0..P), flattened like the module's parameters
template <typename T>
struct RhsCubicMLP {
    static constexpr int D = 2;
    static constexpr int kMaxH = 128;
    static constexpr int kSmem = 2 * kMaxH + kMaxH + 2 * kMaxH + 2;
    static constexpr bool kParams = true;   // 5 H + 2 trainable weights: vjp's parameter sums run in the stage kernel
    static constexpr bool kAutonomous = true;
    static __host__ __device__ __forceinline__ int n_weights(const double *prm) { return (int)prm[0] * 5 + 2; }
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

    // parameter sums: a tile is the block (one row per thread) of (u0, u1, g0, g1); thread x < G H (G = NT / H groups)
    // owns hidden unit h = x % H and walks the rows x / H, x / H + G, ... recomputing z and delta; its accumulators are
    // dW1[0,h], dW1[1,h], db1[h], dW2[h,0], dW2[h,1] and, for h = 0, db2[0], db2[1].  The groups are added in group order.
    static constexpr int kTileVals = 4;
    static constexpr __host__ __device__ int tile_rows(int nt) { return nt; }
    static constexpr __host__ __device__ int acc_count(int) { return 7; }
    static __device__ __forceinline__ void stage(const double *prm, const T * /*sw*/, const T (&y)[2], const T (&g)[2], T *t,
                                                 int ld) {
        const bool cube = prm[1] != 0.0;
        t[0] = cubed(cube, y[0]);
        t[ld] = cubed(cube, y[1]);
        t[2 * ld] = g[0];
        t[3 * ld] = g[1];
    }
    template <int NT>
    static __device__ __forceinline__ void accumulate(const double *prm, const T *sw, const T *tile, const bool *on, double (&acc)[7]) {
        const int H = (int)prm[0], G = NT / H;
        if (threadIdx.x < G * H) {
            const int h = threadIdx.x % H;
            for (int q = threadIdx.x / H; q < NT; q += G) {
                if (!on[q]) continue;
                const T u0 = tile[q], u1 = tile[NT + q];
                const T gq[2] = {tile[2 * NT + q], tile[3 * NT + q]};
                T z, delta;
                unit(sw, H, h, u0, u1, gq, z, delta);
                acc[0] += (double)u0 * (double)delta;
                acc[1] += (double)u1 * (double)delta;
                acc[2] += (double)delta;
                acc[3] += (double)z * (double)gq[0];
                acc[4] += (double)z * (double)gq[1];
                if (h == 0) {
                    acc[5] += (double)gq[0];
                    acc[6] += (double)gq[1];
                }
            }
        }
    }
    template <int NT>
    static __device__ __forceinline__ void partial(const double *prm, const double *red, double *pp) {
        const int H = (int)prm[0], G = NT / H;
        if (threadIdx.x < H) {
            const int h = threadIdx.x;
            double s[7];
#pragma unroll
            for (int q = 0; q < 7; ++q) {
                s[q] = red[q * NT + h];
                for (int gi = 1; gi < G; ++gi) s[q] += red[q * NT + gi * H + h];
            }
            pp[h] = s[0];                                   // W1 (2 x H), b1, W2 (H x 2), b2
            pp[H + h] = s[1];
            pp[2 * H + h] = s[2];
            pp[3 * H + 2 * h] = s[3];
            pp[3 * H + 2 * h + 1] = s[4];
            if (h == 0) {
                pp[5 * H] = s[5];
                pp[5 * H + 1] = s[6];
            }
        }
    }
};

// examples/latent_ode.py:105-120 (LatentODEfunc): fc3(elu(fc2(elu(fc1(z))))), 4 -> H -> H -> 4, H <= 32.  params {H};
// weights staged in shared memory in the module's parameter order, packed
//     [fc1.weight (H x 4) | fc1.bias (H) | fc2.weight (H x H) | fc2.bias (H) | fc3.weight (4 x H) | fc3.bias (4)],
// P = H^2 + 10 H + 4 values.  elu(a) = a > 0 ? a : expm1(a) (torch's F.elu), elu'(a) = a > 0 ? 1 : exp(a) (torch's
// elu_backward).  Every sum runs in index order, the bias added last.  torch evaluates nn.Linear with cuBLAS (its own FMA
// order), so this right-hand side agrees with the module's forward and autograd to rounding, not bit for bit.
template <typename T>
struct RhsLatentMLP {
    static constexpr int D = 4;
    static constexpr int kMaxH = 32;
    static constexpr int kSmem = kMaxH * kMaxH + 10 * kMaxH + 4;
    static constexpr bool kParams = true;
    static constexpr bool kAutonomous = true;
    static __host__ __device__ __forceinline__ int n_weights(const double *prm) {
        const int H = (int)prm[0];
        return H * H + 10 * H + 4;
    }
    static __device__ __forceinline__ float ex(float a) { return expf(a); }
    static __device__ __forceinline__ double ex(double a) { return exp(a); }
    static __device__ __forceinline__ float exm1(float a) { return expm1f(a); }
    static __device__ __forceinline__ double exm1(double a) { return expm1(a); }
    static __device__ __forceinline__ T elu(T a) { return a > T(0) ? a : exm1(a); }
    static __device__ __forceinline__ T elu_d(T a) { return a > T(0) ? T(1) : ex(a); }
    // a1_i = (sum_d y_d W1[i, d]) + b1_i
    static __device__ __forceinline__ T pre1(const T *sw, int H, int i, const T (&y)[4]) {
        using A = Ar<T>;
        const T *w = sw + 4 * i;
        const T s = A::add(A::add(A::add(A::mul(y[0], w[0]), A::mul(y[1], w[1])), A::mul(y[2], w[2])), A::mul(y[3], w[3]));
        return A::add(s, sw[4 * H + i]);
    }
    // The hidden vectors are indexed by runtime loops over H: they live in the thread's local memory (a stack frame of
    // kMaxH or 2 kMaxH values), not in registers -- fully unrolled guarded loops would hold them in registers but multiply
    // the code of every kernel instantiation by kMaxH.
    // z1 = elu(a1)
    static __device__ __forceinline__ void layer1(const T *sw, int H, const T (&y)[4], T (&z1)[kMaxH]) {
#pragma unroll 1
        for (int i = 0; i < H; ++i) z1[i] = elu(pre1(sw, H, i, y));
    }
    // a2_j = (sum_i z1_i W2[j, i]) + b2_j
    static __device__ __forceinline__ T pre2(const T *sw, int H, int j, const T (&z1)[kMaxH]) {
        using A = Ar<T>;
        const T *w = sw + 5 * H + j * H;
        T s = A::mul(z1[0], w[0]);
#pragma unroll 1
        for (int i = 1; i < H; ++i) s = A::add(s, A::mul(z1[i], w[i]));
        return A::add(s, sw[5 * H + H * H + j]);
    }
    // (W3^T g)_j = sum_d W3[d, j] g_d
    static __device__ __forceinline__ T back3(const T *W3, int H, int j, const T (&g)[4]) {
        using A = Ar<T>;
        return A::add(A::add(A::add(A::mul(W3[j], g[0]), A::mul(W3[H + j], g[1])), A::mul(W3[2 * H + j], g[2])), A::mul(W3[3 * H + j], g[3]));
    }
    static __device__ __forceinline__ void eval(const double *prm, const T *sw, T /*t*/, const T (&y)[4], T (&dy)[4]) {
        using A = Ar<T>;
        const int H = (int)prm[0];
        const T *W3 = sw + 6 * H + H * H, *b3 = W3 + 4 * H;
        T z1[kMaxH];
        layer1(sw, H, y, z1);
        T o[4] = {T(0), T(0), T(0), T(0)};
#pragma unroll 1
        for (int j = 0; j < H; ++j) {                    // layer 2 streamed one output unit at a time into layer 3
            const T z2 = elu(pre2(sw, H, j, z1));
#pragma unroll
            for (int d = 0; d < 4; ++d) o[d] = A::add(o[d], A::mul(z2, W3[d * H + j]));
        }
#pragma unroll
        for (int d = 0; d < 4; ++d) dy[d] = A::add(o[d], b3[d]);
    }
    // f(y) and gy = W1^T delta1 with delta2 = (W3^T g) elu'(a2), delta1 = (W2^T delta2) elu'(a1)
    static __device__ __forceinline__ void vjp(const double *prm, const T *sw, T /*t*/, const T (&y)[4], const T (&g)[4],
                                               T (&f)[4], T (&gy)[4]) {
        using A = Ar<T>;
        const int H = (int)prm[0];
        const T *W2 = sw + 5 * H, *W3 = sw + 6 * H + H * H, *b3 = W3 + 4 * H;
        T z1[kMaxH], s[kMaxH];
        layer1(sw, H, y, z1);
#pragma unroll 1
        for (int i = 0; i < H; ++i) s[i] = T(0);
        T o[4] = {T(0), T(0), T(0), T(0)};
#pragma unroll 1
        for (int j = 0; j < H; ++j) {
            const T a2 = pre2(sw, H, j, z1);
            const T z2 = elu(a2);
#pragma unroll
            for (int d = 0; d < 4; ++d) o[d] = A::add(o[d], A::mul(z2, W3[d * H + j]));
            const T d2 = A::mul(back3(W3, H, j, g), elu_d(a2));
#pragma unroll 1
            for (int i = 0; i < H; ++i) s[i] = A::add(s[i], A::mul(W2[j * H + i], d2));
        }
#pragma unroll
        for (int d = 0; d < 4; ++d) {
            f[d] = A::add(o[d], b3[d]);
            gy[d] = T(0);
        }
#pragma unroll 1
        for (int i = 0; i < H; ++i) {
            const T d1 = A::mul(s[i], elu_d(pre1(sw, H, i, y)));
#pragma unroll
            for (int d = 0; d < 4; ++d) gy[d] = A::add(gy[d], A::mul(sw[4 * i + d], d1));
        }
    }

    // parameter sums: a tile of tile_rows rows holds, per row, [y (4) | z1 (H) | z2 (H) | g (4) | delta1 (H) | delta2 (H)]
    // (8 + 4 H values, vjp's arithmetic).  Every weight is a sum over rows of one product of two of them (a bias: of one):
    // thread x owns the flattened parameters x, x + NT, x + 2 NT, ..., so a block's partial needs no combine.
    static constexpr int kTileVals = 8 + 4 * kMaxH;
    static __device__ __forceinline__ int tile_vals(const double *prm) { return 8 + 4 * (int)prm[0]; }
    static constexpr __host__ __device__ int tile_rows(int nt) { return (sizeof(T) == 8 ? 16 : 32) < nt ? (sizeof(T) == 8 ? 16 : 32) : nt; }
    static constexpr __host__ __device__ int acc_count(int nt) { return (kSmem + nt - 1) / nt; }
    static __device__ __forceinline__ void stage(const double *prm, const T *sw, const T (&y)[4], const T (&g)[4], T *t, int ld) {
        using A = Ar<T>;
        const int H = (int)prm[0];
        const T *W2 = sw + 5 * H, *W3 = sw + 6 * H + H * H;
        T *z1 = t + 4 * ld, *z2 = t + (4 + H) * ld, *d1 = t + (8 + 2 * H) * ld, *d2 = t + (8 + 3 * H) * ld;
#pragma unroll
        for (int d = 0; d < 4; ++d) {
            t[d * ld] = y[d];
            t[(4 + 2 * H + d) * ld] = g[d];
        }
#pragma unroll 1
        for (int i = 0; i < H; ++i) z1[i * ld] = elu(pre1(sw, H, i, y));
#pragma unroll 1
        for (int j = 0; j < H; ++j) {
            T a = A::mul(z1[0], W2[j * H]);
#pragma unroll 1
            for (int i = 1; i < H; ++i) a = A::add(a, A::mul(z1[i * ld], W2[j * H + i]));
            a = A::add(a, sw[5 * H + H * H + j]);
            z2[j * ld] = elu(a);
            d2[j * ld] = A::mul(back3(W3, H, j, g), elu_d(a));
        }
#pragma unroll 1
        for (int i = 0; i < H; ++i) {
            T s = T(0);
#pragma unroll 1
            for (int j = 0; j < H; ++j) s = A::add(s, A::mul(W2[j * H + i], d2[j * ld]));
            d1[i * ld] = A::mul(s, elu_d(pre1(sw, H, i, y)));
        }
    }
    // tile value indices (a, b) of flattened parameter q: its per-row term is v_a v_b, or v_a for a bias (b < 0)
    static __device__ __forceinline__ void term(int H, int q, int &a, int &b) {
        const int z1 = 4, z2 = 4 + H, g = 4 + 2 * H, d1 = 8 + 2 * H, d2 = 8 + 3 * H;
        if (q < 4 * H) { a = d1 + q / 4; b = q % 4; return; }                              // fc1.weight[j, d]
        q -= 4 * H;
        if (q < H) { a = d1 + q; b = -1; return; }                                         // fc1.bias[j]
        q -= H;
        if (q < H * H) { a = d2 + q / H; b = z1 + q % H; return; }                        // fc2.weight[j, i]
        q -= H * H;
        if (q < H) { a = d2 + q; b = -1; return; }                                         // fc2.bias[j]
        q -= H;
        if (q < 4 * H) { a = g + q / H; b = z2 + q % H; return; }                          // fc3.weight[d, j]
        a = g + (q - 4 * H);                                                               // fc3.bias[d]
        b = -1;
    }
    template <int NT, int NA>
    static __device__ __forceinline__ void accumulate(const double *prm, const T * /*sw*/, const T *tile, const bool *on,
                                                      double (&acc)[NA]) {
        constexpr int R = tile_rows(NT);
        const int H = (int)prm[0], P = n_weights(prm);
#pragma unroll
        for (int k = 0; k < NA; ++k) {
            const int q = threadIdx.x + k * NT;
            if (q < P) {
                int a, b;
                term(H, q, a, b);
                const T *va = tile + a * R, *vb = tile + (b < 0 ? 0 : b) * R;
#pragma unroll 4
                for (int r = 0; r < R; ++r) {
                    if (!on[r]) continue;
                    acc[k] += b < 0 ? (double)va[r] : (double)va[r] * (double)vb[r];
                }
            }
        }
    }
    template <int NT>
    static __device__ __forceinline__ void partial(const double *prm, const double *red, double *pp) {
        const int P = n_weights(prm);
#pragma unroll
        for (int k = 0; k < acc_count(NT); ++k) {
            const int q = threadIdx.x + k * NT;
            if (q < P) pp[q] = red[k * NT + threadIdx.x];
        }
    }
};

// ------------------------------------------------------------------------------------------------
// the parameter sums of the kernels above, on RHS's hooks.  The order is fixed: rows in tile order, the hooks' unit
// order, then (par_last_block) the block partials in block order -- the result depends on the grid, never on timing, and
// no floating-point atomics are involved.
// ------------------------------------------------------------------------------------------------
// staged weights: sw[0..n_weights) of the right-hand side's data, for RHS with weights (kSmem > 1); ends with a barrier
template <typename T, typename RHS>
__device__ __forceinline__ void stage_weights(const double *prm, const void *data, T *sw, int nthreads) {
    if constexpr (RHS::kSmem > 1) {
        const int nw = RHS::n_weights(prm);
        for (int q = threadIdx.x; q < nw && q < RHS::kSmem; q += nthreads) sw[q] = ((const T *)data)[q];
        __syncthreads();
    }
}

// Shared-memory sizes (in elements) of the parameter sums of RHS in a block of NT threads
template <typename T, typename RHS, int NT, bool PAR>
struct ParShape {
    static constexpr int rows = 1, tile = 1, acc = 1, red = 1;
};
template <typename T, typename RHS, int NT>
struct ParShape<T, RHS, NT, true> {
    static constexpr int rows = RHS::tile_rows(NT);
    static constexpr int tile = RHS::kTileVals * rows;
    static constexpr int acc = RHS::acc_count(NT);
    static constexpr int red = acc * NT;
};

// One chunk of NT rows, thread x holding row x (on: the row contributes): the chunk is staged tile by tile and each tile
// added to the accumulators.  Every thread of the block calls it.
template <typename T, typename RHS, int NT, int NA>
__device__ __forceinline__ void par_tiles(const double *prm, const T *sw, T *tile, bool *on_s, bool on, const T (&y)[RHS::D],
                                          const T (&g)[RHS::D], double (&acc)[NA]) {
    constexpr int R = RHS::tile_rows(NT);
    static_assert(NT % R == 0 && NA == RHS::acc_count(NT), "tile rows divide the block; one accumulator set per thread");
    if constexpr (R == NT) {                 // one tile: every thread stages its own row
        if (on) RHS::stage(prm, sw, y, g, tile + threadIdx.x, NT);
        on_s[threadIdx.x] = on;
        __syncthreads();
        RHS::template accumulate<NT>(prm, sw, tile, on_s, acc);
        __syncthreads();
    } else {
        // every thread forms its row's values at once (in its stack frame); the tiles then only copy them, in turn
        T v[RHS::kTileVals];
        if (on) RHS::stage(prm, sw, y, g, v, 1);
        const int nv = RHS::tile_vals(prm);
        for (int s = 0; s < NT / R; ++s) {
            if ((int)threadIdx.x / R == s) {
                const int q = threadIdx.x % R;
                if (on)
                    for (int k = 0; k < nv; ++k) tile[k * R + q] = v[k];
                on_s[q] = on;
            }
            __syncthreads();
            RHS::template accumulate<NT>(prm, sw, tile, on_s, acc);
            __syncthreads();
        }
    }
}

// the block's partial pp[0..P) from every thread's accumulators (red: ParShape::red doubles of shared memory)
template <typename RHS, int NT, int NA>
__device__ __forceinline__ void par_block_partial(const double *prm, const double (&acc)[NA], double *red, double *pp) {
#pragma unroll
    for (int q = 0; q < NA; ++q) red[q * NT + threadIdx.x] = acc[q];
    __syncthreads();
    RHS::template partial<NT>(prm, red, pp);
}

// the last block to arrive sums the block partials part[b][0..P) in block order, hands each sum to put(q, s) and resets
// the ticket
template <int NT, typename F>
__device__ __forceinline__ void par_last_block(unsigned *ticket, const double *part, int P, F &&put) {
    if (!last_block_arrives(ticket)) return;
    for (int q = threadIdx.x; q < P; q += NT) {
        double s = 0.0;
        for (unsigned b = 0; b < gridDim.x; ++b) s += __ldcg(part + (size_t)b * P + q);
        put(q, s);
    }
    if (threadIdx.x == 0) *ticket = 0;
}


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
        case B2ODE_RHS_LATENT_MLP: return RhsLatentMLP<double>::D;
    }
    return -1;
}

// P, the trainable weights of a validated description (0 for the systems without any)
static inline int rhs_n_weights(const b2ode_rhs_desc *r) {
    switch (r->kind) {
        case B2ODE_RHS_CUBIC_MLP: return RhsCubicMLP<double>::n_weights(r->params);
        case B2ODE_RHS_LATENT_MLP: return RhsLatentMLP<double>::n_weights(r->params);
    }
    return 0;
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
    if (r->kind == B2ODE_RHS_LATENT_MLP &&
        (!r->data || r->n_params < 1 || !(r->params[0] >= 1 && r->params[0] <= RhsLatentMLP<double>::kMaxH)))
        return b2_fail(B2ODE_EINVAL, "latent-MLP right-hand side needs {H in [1, 32]} and its weights");
    *rows = n_elems / D;
    return 0;
}

// odeint_adjoint's augmented state for a built-in right-hand side (tfdiffeq/adjoint.py:146): four segments (y, adj_y,
// adj_t, adj_params) of (N, N, 1, max(P, 1)) elements, where P = rhs_n_weights (5 H + 2 for a B2ODE_RHS_CUBIC_MLP,
// H^2 + 10 H + 4 for a B2ODE_RHS_LATENT_MLP) when the weights are all trainable and 0 otherwise (adj_params is then the
// 0-dim zero).  Validates `r` and the layout and sets *rows = N / D and
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
    if (r->kind == B2ODE_RHS_CUBIC_MLP || r->kind == B2ODE_RHS_LATENT_MLP) {
        const int H = (int)r->params[0], nw = rhs_n_weights(r);
        if (seg_len[3] != 1 && seg_len[3] != nw)
            return b2_fail(B2ODE_EINVAL, "adj_params has %lld elements: a %s of hidden width %d takes 1 (frozen weights) or %d",
                           (long long)seg_len[3], r->kind == B2ODE_RHS_CUBIC_MLP ? "cubic-MLP" : "latent-MLP", H, nw);
        P = seg_len[3] == 1 ? 0 : nw;
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
        case B2ODE_RHS_LATENT_MLP: return f(RhsLatentMLP<T>());
    }
    return b2_fail(B2ODE_EINVAL, "unknown built-in right-hand side %d", kind);
}
