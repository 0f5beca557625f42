// b2ode_dev.cuh -- device helpers shared by b2ode.cu (generic func path) and b2ode_fused.cu (built-in RHS).
#pragma once
#include "b2ode.h"
#include "b2ode_pay16.cuh"

#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <new>
#include <type_traits>
#include <utility>

static_assert(sizeof(b2ode_state) == 256, "b2ode_state must stay 256 bytes");

// ------------------------------------------------------------------------------------------------
// host-side error plumbing
// ------------------------------------------------------------------------------------------------
int b2_fail(int code, const char *fmt, ...);      // defined in b2ode.cu; records the thread-local error string
void b2_count_launch(void);                     // bench.py's gpu_launches counter (b2ode.cu)
int b2_timing_begin(int fam, cudaStream_t st);  // optional CUDA-event timing of a kernel family (b2ode.cu)
void b2_timing_end(int fam, int slot, cudaStream_t st);

#define B2_CUDA(x)                                                                         \
    do {                                                                                   \
        cudaError_t e_ = (x);                                                              \
        if (e_ != cudaSuccess) return b2_fail((int)e_, "%s -> %s", #x, cudaGetErrorString(e_)); \
    } while (0)

// f(std::integral_constant<int, N>{}) for the N in Ns equal to n: the one switch from a runtime count to a template argument.
// Any other n fails with B2ODE_EINVAL and the message fmt formats from args.
template <int... Ns, typename F, typename... Args>
static int dispatch_count(std::integer_sequence<int, Ns...>, int n, F &&f, const char *fmt, Args... args) {
    int rc = 0;
    if (((n == Ns && ((rc = f(std::integral_constant<int, Ns>{})), true)) || ...)) return rc;
    return b2_fail(B2ODE_EINVAL, fmt, args...);
}

// Grid of a static grid-stride launch: one block per `threads` rows, at least one, at most blocks_per_sm per SM (132 SMs
// when sm_count is not given).  Workspace sizes derive from it, so it depends on the batch and sm_count only.
static inline long long capped_grid(long long rows, int threads, int blocks_per_sm, int sm_count) {
    const long long need = (rows + threads - 1) / threads;
    const long long cap = (long long)(sm_count > 0 ? sm_count : 132) * blocks_per_sm;
    return need < cap ? (need < 1 ? 1 : need) : cap;
}

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

template <typename T>
struct Ar;
template <>
struct Ar<double> {
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
    static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
    static __device__ __forceinline__ double abs(double a) { return fabs(a); }
    static __device__ __forceinline__ double sqrt(double a) { return __dsqrt_rn(a); }
    static __device__ __forceinline__ double pow(double a, double b) { return ::pow(a, b); }
};
template <>
struct Ar<float> {
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
    static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
    static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
    static __device__ __forceinline__ float abs(float a) { return fabsf(a); }
    static __device__ __forceinline__ float sqrt(float a) { return __fsqrt_rn(a); }
    static __device__ __forceinline__ float pow(float a, float b) { return ::powf(a, b); }
};

// V elements of T; V*sizeof(T) is 16 (vector path) or sizeof(T) (scalar path)
template <typename T, int V>
struct alignas(sizeof(T) * V) Pack {
    T v[V];
};

template <typename T, int V>
__device__ __forceinline__ Pack<T, V> ld_pack(const T *p, long long i) {
    Pack<T, V> r;
    if constexpr (V == 1) {
        r.v[0] = p[i];
    } else {
        static_assert(sizeof(T) * V == 16, "vector path is 16 bytes");
        *reinterpret_cast<int4 *>(&r) = *reinterpret_cast<const int4 *>(p + i * V);
    }
    return r;
}

template <typename T, int V>
__device__ __forceinline__ void st_pack(T *p, long long i, const Pack<T, V> &r) {
    if constexpr (V == 1) {
        p[i] = r.v[0];
    } else {
        *reinterpret_cast<int4 *>(p + i * V) = *reinterpret_cast<const int4 *>(&r);
    }
}

// geometry of a launch: blocks [blk_begin[s], blk_begin[s+1]) work on segment s
struct SegGeom {
    int nseg;
    int blk_begin[B2ODE_MAXSEG + 1];
    long long n[B2ODE_MAXSEG];
    unsigned vec_mask;  // bit s: every pointer of segment s is 16-byte aligned
};

__device__ __forceinline__ int find_seg(const SegGeom &g, int b) {
    int s = 0;
    while (s + 1 < g.nseg && b >= g.blk_begin[s + 1]) ++s;
    return s;
}

template <int V>
using IC = std::integral_constant<int, V>;

// Run body(IC<V>, pack_index) over one segment: 16-byte packs + scalar tail, or all-scalar.
template <typename T, typename F>
__device__ __forceinline__ void seg_for_each(long long n, bool vec_ok, int bl, int nb, F &&body) {
    constexpr int VW = 16 / sizeof(T);
    const long long stride = (long long)nb * kThreads;
    const long long first = (long long)bl * kThreads + threadIdx.x;
    if (vec_ok) {
        const long long nv = n / VW;
#pragma unroll 1
        for (long long i = first; i < nv; i += stride) body(IC<VW>{}, i);
        const long long tail = nv * VW + threadIdx.x;
        if (bl == 0 && tail < n) body(IC<1>{}, tail);
    } else {
        for (long long i = first; i < n; i += stride) body(IC<1>{}, i);
    }
}

// One record per block, written once, reduced by the last block in block order.  Four columns; the
// template mask MM says which columns combine with a NaN-propagating max (bit set) instead of a sum.
struct Partial {
    double v[4];
};

__device__ __forceinline__ double nan_max(double a, double b) { return (a != a || b != b) ? (double)NAN : fmax(a, b); }
__device__ __forceinline__ double nan_min(double a, double b) { return (a != a || b != b) ? (double)NAN : fmin(a, b); }

template <unsigned MM>
__device__ __forceinline__ Partial combine(const Partial &a, const Partial &b) {
    Partial r;
#pragma unroll
    for (int c = 0; c < 4; ++c) r.v[c] = ((MM >> c) & 1u) ? nan_max(a.v[c], b.v[c]) : a.v[c] + b.v[c];
    return r;
}

template <unsigned MM>
__device__ __forceinline__ Partial identity() {
    Partial r;
#pragma unroll
    for (int c = 0; c < 4; ++c) r.v[c] = 0.0;   // sums start at 0; the maxima are of absolute values (>= 0)
    return r;
}

// block-wide reduction, fixed order (xor butterfly inside a warp, then warps 0..7); result valid in thread 0
template <unsigned MM>
__device__ __forceinline__ Partial block_reduce(Partial x) {
    __shared__ Partial sh[kWarps];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Partial y;
#pragma unroll
        for (int c = 0; c < 4; ++c) y.v[c] = __shfl_xor_sync(0xffffffffu, x.v[c], o);
        x = combine<MM>(x, y);
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();   // protect sh[] against a previous use
    if (l == 0) sh[w] = x;
    __syncthreads();
    Partial r = identity<MM>();
    if (threadIdx.x == 0) {
        r = sh[0];
        for (int i = 1; i < kWarps; ++i) r = combine<MM>(r, sh[i]);
    }
    return r;
}

// NaN-aware abs-max accumulation: fmax() drops NaN, so NaN is tracked separately and re-injected.
template <typename T>
struct AbsMax {
    T mx = T(0);
    bool nan = false;
    __device__ __forceinline__ void see(T v) {
        T a = Ar<T>::abs(v);
        nan |= (a != a);
        mx = (a > mx) ? a : mx;
    }
    __device__ __forceinline__ double value() const { return nan ? (double)NAN : (double)mx; }
};

// returns true in every thread of exactly one block: the last one to arrive
__device__ __forceinline__ bool last_block_arrives(unsigned *ticket) {
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned t = atomicAdd(ticket, 1u);
        is_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (is_last) __threadfence();
    return is_last;
}

// ------------------------------------------------------------------------------------------------
// cross-GPU exchange of the per-segment partials (shared-step groups; new, SURVEY 8e)
// ------------------------------------------------------------------------------------------------
struct MailSlot {
    double vals[B2ODE_MAXSEG][4];
    unsigned long long seq;
    unsigned long long pad[7];
};
constexpr int kMaxFusedBlocks = 320;     // blocks of one rank's persistent fused kernel (H100: 132 SMs x 2 blocks, with headroom)
struct Mailbox {
    MailSlot slot[2][B2ODE_MAXPEERS];
    unsigned long long local_seq;   // exchanges completed by the owning rank; persists across solves
    unsigned long long ll_seq;      // exchanges of the persistent fused kernel so far; persists across solves
    unsigned fused_hw[2];           // per buffer parity: how many slots of THIS rank's region in its peers' mailboxes hold
                                    // partials (= the grid of the last solve that wrote that buffer); slots beyond are poison
    unsigned long long pad[5];
    // receive area of the persistent fused kernel (b2ode_fused.cu): every block of rank s stores its 16-byte tagged partial
    // of exchange `seq` into fused_part[seq & 1][s][block] of every other rank's mailbox (plain NVLink stores, no atomics)
    // A slot that holds no partial holds the POISON pattern {tag 0, tag 1}, which no exchange number validates: mailboxes are
    // created poisoned, and a solve with a smaller grid than its predecessor poisons the slots it no longer writes (before its
    // first exchange on each buffer), so a later, larger solve can never mistake an old partial with a matching tag for a
    // fresh one.
    unsigned long long fused_part[2][B2ODE_MAXPEERS][kMaxFusedBlocks][2];
};
constexpr unsigned long long kPoisonW0 = kPayPoisonW0, kPoisonW1 = kPayPoisonW1;   // b2ode_pay16.cuh

struct CommParams {
    int rank;
    int nranks;  // 0 or 1: no exchange
    unsigned repl_mask;   // bit s: segment s is replicated (bit-identical on every rank): its totals are NOT combined
    Mailbox *box[B2ODE_MAXPEERS];
    int grid_of[B2ODE_MAXPEERS];   // blocks of rank r's persistent fused kernel (fused path only)
};

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double ld_relaxed_sys(const double *p) {
    double v;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys(double *p, double v) {
    asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}

// Called by ALL threads of the last block.  tot[s] (shared memory, [nseg]) holds this rank's totals on
// entry and the group totals (combined in rank order: deterministic and identical on every rank) on exit.
template <unsigned MM>
__device__ void group_combine(const CommParams &cp, b2ode_state *st, Partial *tot, int nseg) {
    if (cp.nranks <= 1) return;
    __shared__ unsigned long long seq_sh;
    if (threadIdx.x == 0) seq_sh = cp.box[cp.rank]->local_seq + 1;
    __syncthreads();
    const unsigned long long seq = seq_sh;
    const int par = (int)(seq & 1ull);
    if (threadIdx.x < cp.nranks) {
        // push my totals into peer q's mailbox, slot [par][my rank], then release the sequence number
        const int q = threadIdx.x;
        MailSlot *dst = &cp.box[q]->slot[par][cp.rank];
        for (int s = 0; s < nseg; ++s)
            for (int c = 0; c < 4; ++c) st_relaxed_sys(&dst->vals[s][c], tot[s].v[c]);
        __threadfence_system();
        st_release_sys(&dst->seq, seq);
        // wait for rank q's totals in MY mailbox
        const MailSlot *src = &cp.box[cp.rank]->slot[par][q];
        while (ld_acquire_sys(&src->seq) != seq) __nanosleep(20);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const Mailbox *mine = cp.box[cp.rank];
        for (int s = 0; s < nseg; ++s) {
            if ((cp.repl_mask >> s) & 1u) continue;      // every rank already holds the whole segment
            Partial p = identity<MM>();
            for (int q = 0; q < cp.nranks; ++q) {
                const MailSlot *src = &mine->slot[par][q];
                Partial x;
                for (int c = 0; c < 4; ++c) x.v[c] = ld_relaxed_sys(&src->vals[s][c]);
                p = (q == 0) ? x : combine<MM>(p, x);
            }
            tot[s] = p;
        }
        cp.box[cp.rank]->local_seq = seq;
        st->xseq = seq;
    }
    __syncthreads();
}

// Last block: reduce the per-block partials of every segment in block order into tot[] (shared).
template <unsigned MM>
__device__ void reduce_partials(const SegGeom &g, const Partial *part, Partial *tot) {
    for (int s = 0; s < g.nseg; ++s) {
        Partial acc = identity<MM>();
        for (int b = g.blk_begin[s] + threadIdx.x; b < g.blk_begin[s + 1]; b += kThreads) acc = combine<MM>(acc, part[b]);
        Partial r = block_reduce<MM>(acc);
        if (threadIdx.x == 0) tot[s] = r;
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// controller parameters shared by the kernels that end an attempt / the initial step
// ------------------------------------------------------------------------------------------------
struct CtrlParams {
    int n_k;                      // s
    int controller;               // B2ODE_CTRL_*
    double alpha[B2ODE_MAXK];     // s-1 entries
    double rtol[B2ODE_MAXSEG], atol[B2ODE_MAXSEG];
    double safety, ifactor, dfactor, exponent;
    double inv_safety, inv_ifactor, inv_dfactor;   // host-computed reciprocals (the controller is a serial latency chain)
    long long max_num_steps;
    int init_order;
    int n_out;
    const double *t_out;
    void *tstage;                 // n_k scalars of the state dtype
    long long n_global[B2ODE_MAXSEG];   // element count of the segment over the whole shared-step group
};

// Copies the controller's part of a descriptor, every rtol / atol entry included: ctrl_decide, init_h0 and init_dt read only
// the segments they are given, so entries past a caller's segment count are never read.  The caller sets n_out, t_out,
// tstage and n_global.
static inline void fill_ctrl(CtrlParams &c, const b2ode_adaptive_desc &d) {
    c.n_k = d.n_k;
    c.controller = d.controller;
    for (int i = 0; i < B2ODE_MAXK; ++i) c.alpha[i] = d.alpha[i];
    for (int i = 0; i < B2ODE_MAXSEG; ++i) {
        c.rtol[i] = d.rtol[i];
        c.atol[i] = d.atol[i];
    }
    c.safety = d.safety;
    c.ifactor = d.ifactor;
    c.dfactor = d.dfactor;
    c.exponent = d.exponent;
    c.inv_safety = 1.0 / d.safety;
    c.inv_ifactor = 1.0 / d.ifactor;
    c.inv_dfactor = 1.0 / d.dfactor;
    c.max_num_steps = d.max_num_steps;
    c.init_order = d.init_order;
}

// rk_common.py:45-50: t0 and dt are cast to the state dtype, ti = t0 + alpha_i * dt in that dtype
template <typename T>
__device__ void write_stage_times(const CtrlParams &c, double t_cur, double dt) {
    T *ts = reinterpret_cast<T *>(c.tstage);
    const T t0 = (T)t_cur, d = (T)dt;
    for (int i = 0; i + 1 < c.n_k; ++i) ts[i] = Ar<T>::add(t0, Ar<T>::mul((T)c.alpha[i], d));
}

// misc.py:250-264 (error ratio per segment, ONE scalar tolerance per segment :257), dopri5.py:108 (accept iff
// every segment passes) and misc.py:267-287 / tsit5.py:53-62 (next step size).  Pure function of the group
// totals, so every rank / every thread that evaluates it gets bit-identical decisions.
struct CtrlDecision {
    bool accept;
    bool bad0;       // non-finite value in y0 (dopri5.py:100)
    double m;        // max (or pooled) mean-square error ratio
    double dt_next;
};

// The controller runs once per attempted step on the critical path of EVERY attempt (one thread, all other threads of the
// GPU waiting), so its dependent-latency chain is kept short: one division for the error ratio (sum err^2 / (tol^2 * n)
// instead of two), x**e as exp2(e * log2(x)) instead of pow(), reciprocals of safety / ifactor / dfactor precomputed on
// the host.  dt_next's relative error against a correctly rounded evaluation of the reference's `sqrt(m) ** e / safety`
// at the same m is bounded in tests/controller_cases.py (dt_bound): 3 ln2 2^-53 |e log2 sqrt(m)| from log2 (1 ulp) and the
// multiply by e, plus 4 2^-53 from exp2 (2 ulp), 2 2^-53 from 1/safety and its multiply, one for the final division, and
// the ratio's own error scaled by e/2 -- about 1e-15 for the probes there, far inside the 1e-6 / 1e-3 parity bars (dt is
// a free parameter of the method; the accept decision is unaffected).  The clamps divide by the host's fp64 1/ifactor
// and 1/dfactor, as the reference does, and are correctly rounded.
template <typename T>
__device__ __forceinline__ CtrlDecision ctrl_decide(const CtrlParams &c, const Partial *tot, int nseg, double dt) {
    bool accept = true;
    double m = 0.0;
    double pooled = 0.0;
    long long pooled_n = 0;
    bool bad0 = false;
    for (int s = 0; s < nseg; ++s) {
        bad0 |= (tot[s].v[3] > 0.0);
        // tol = atol + rtol * reduce_max([|y0|, |y1|]): ONE scalar per segment (misc.py:257)
        const double mm = nan_max(tot[s].v[1], tot[s].v[2]);
        const T tol = Ar<T>::add((T)c.atol[s], Ar<T>::mul((T)c.rtol[s], (T)mm));
        const double tol2 = (double)tol * (double)tol;
        if (c.controller == B2ODE_CTRL_TSIT5) {
            pooled += tot[s].v[0] / tol2;
            pooled_n += c.n_global[s];
        } else {
            // mean((err / tol)^2) as sum(err^2) / (tol^2 * n): a one-pass global-tolerance form of misc.py:259-263
            const T msr = (T)(tot[s].v[0] / (tol2 * (double)c.n_global[s]));
            accept = accept && (msr <= T(1));
            m = (s == 0) ? (double)msr : nan_max(m, (double)msr);
        }
    }
    if (c.controller == B2ODE_CTRL_TSIT5) {
        const T msr = (T)(pooled / (double)pooled_n);
        accept = (msr <= T(1));
        m = (double)msr;
    }
    // _optimal_step_size
    double dt_next;
    if (m == 0.0) {
        dt_next = dt * c.ifactor;
    } else {
        const double inv_df = (m < 1.0) ? 1.0 : c.inv_dfactor;
        const double er = (c.controller == B2ODE_CTRL_TSIT5) ? m : (double)Ar<T>::sqrt((T)m);
        const double cand = exp2(c.exponent * log2(er)) * c.inv_safety;
        const double factor = nan_max(c.inv_ifactor, nan_min(cand, inv_df));
        dt_next = dt / factor;
    }
    CtrlDecision d;
    d.accept = accept;
    d.bad0 = bad0;
    d.m = m;
    d.dt_next = dt_next;
    return d;
}

// dopri5.py:98: the step no longer moves t (a NaN dt lands here too)
__device__ __forceinline__ bool step_underflows(double t, double dt) { return !(t + dt > t); }

// advance(): the first output index at or after `cur` whose time lies beyond t1 (`while next_t > t1`)
__device__ __forceinline__ int next_cursor(const double *__restrict__ t_out, int cur, int n_out, double t1) {
    int c2 = cur;
    while (c2 < n_out && __ldg(t_out + c2) <= t1) ++c2;
    return c2;
}

// What an attempt's decision does to the solve (dopri5.py:83-120): status bits, whether the step advances the solution,
// the new t1, output cursor and count of steps without progress, and whether the solve ends.  c2 is the cursor the
// accepted step would reach (next_cursor from cur at t_cur + dt).
struct StepAdvance {
    unsigned status;
    bool adv;
    double t1;
    int cur;
    long long nadv;
    bool done;
};

__device__ __forceinline__ StepAdvance advance_step(const CtrlDecision &dec, unsigned status, int cur, int c2, int n_out,
                                                    long long nadv, long long max_num_steps, double t_cur, double dt) {
    StepAdvance a;
    a.status = status;
    if (dec.bad0) a.status |= B2ODE_ST_NONFINITE;                    // the reference asserts this before taking the step
    a.adv = dec.accept && !dec.bad0;
    a.t1 = dec.accept ? t_cur + dt : t_cur;
    a.cur = a.adv ? c2 : cur;
    a.nadv = (a.cur > cur) ? 0 : nadv + 1;
    a.done = a.cur >= n_out;
    if (!a.done) {
        if (a.nadv >= max_num_steps) a.status |= B2ODE_ST_MAXSTEPS;  // dopri5.py:85
        if (step_underflows(a.t1, dec.dt_next)) a.status |= B2ODE_ST_UNDERFLOW;
    }
    if (a.status) a.done = true;
    return a;
}

// misc.py:226-234: d0, d1 (RMS norms from the sums of squares in columns 0 and 1) and the first guess h0
template <typename T>
__device__ __forceinline__ T init_h0(const CtrlParams &c, const Partial *tot, int nseg, T *d1max_out) {
    T d0max = T(0), d1max = T(0), ratio = T(0);
    bool first = true;
    for (int sg = 0; sg < nseg; ++sg) {
        const T rn = Ar<T>::sqrt((T)(double)c.n_global[sg]);               // numel ** 0.5, misc.py:173
        const T d0 = Ar<T>::div((T)sqrt(tot[sg].v[0]), rn), d1 = Ar<T>::div((T)sqrt(tot[sg].v[1]), rn);
        const T q = Ar<T>::div(d0, d1);
        if (first) {
            d0max = d0;
            d1max = d1;
            ratio = q;
            first = false;
        } else {
            d0max = (d0 > d0max) ? d0 : d0max;     // python max(): keeps the first unless strictly greater
            d1max = (d1 > d1max) ? d1 : d1max;
            ratio = (q > ratio) ? q : ratio;
        }
    }
    T h0;
    if ((double)d0max < 1e-5 || (double)d1max < 1e-5) h0 = (T)1e-6;           // misc.py:231-232
    else h0 = Ar<T>::mul((T)0.01, ratio);                                     // misc.py:234
    *d1max_out = d1max;
    return h0;
}

// misc.py:238-247: d2 from the sum of squares in column 0, h1, and the first step min(100 h0, h1)
template <typename T>
__device__ __forceinline__ T init_dt(const CtrlParams &c, const Partial *tot, int nseg, T h0, T d1max) {
    T d2max = T(0);
    for (int sg = 0; sg < nseg; ++sg) {
        const T rn = Ar<T>::sqrt((T)(double)c.n_global[sg]);
        const T d2 = Ar<T>::div(Ar<T>::div((T)sqrt(tot[sg].v[0]), rn), h0);
        d2max = (sg == 0 || d2 > d2max) ? d2 : d2max;
    }
    T h1;
    if ((double)d1max <= 1e-15 && (double)d2max <= 1e-15) {
        const T alt = Ar<T>::mul(h0, (T)1e-3);
        h1 = ((T)1e-6 > alt) ? (T)1e-6 : alt;                                 // misc.py:242-243
    } else {
        const T mx = (d2max > d1max) ? d2max : d1max;                         // max(d1 + d2): tuple concat
        h1 = Ar<T>::pow(Ar<T>::div((T)0.01, mx), (T)(1.0 / (double)(c.init_order + 1)));   // misc.py:245
    }
    const T h100 = Ar<T>::mul(T(100), h0);
    return (h1 < h100) ? h1 : h100;                                           // misc.py:247
}

// ------------------------------------------------------------------------------------------------
// dense output: the quartic fit of one accepted step (interp.py:22-67)
// ------------------------------------------------------------------------------------------------
// Coefficients of the fit that are the same for every element: dt * c_mid[j] and the five multiples of dt of the fit
// (-2, 2, 5, -3, -4).  Every one multiplies a k, so in the fused kernels dt carries the sign of the time direction (see `rhs`
// in k_fused_adaptive).
template <typename T, int S>
struct DenseConst {
    T cmid[S];
    T fc[5];
};

template <typename T>
__device__ __forceinline__ T fit_coef(int q) { return q == 0 ? T(-2) : q == 1 ? T(2) : q == 2 ? T(5) : q == 3 ? T(-3) : T(-4); }

// The quartic fit of one element (interp.py:22-36, python sum() left to right) from the step's first and last k (f0, f1),
// its ends (y0, y1) and the midpoint value ymid: x^4, x^3, x^2 and x coefficients ca, cb, cc, cd.  dtk is dt with the sign
// of the k's.
template <typename T, int S>
__device__ __forceinline__ void quartic_fit(const DenseConst<T, S> &dc, T dtk, T f0, T f1, T y0, T y1, T ymid, T &ca, T &cb,
                                            T &cc, T &cd) {
    using A = Ar<T>;
    T a = A::mul(dc.fc[0], f0);
    a = A::add(a, A::mul(dc.fc[1], f1));
    a = A::add(a, A::mul(T(-8), y0));
    a = A::add(a, A::mul(T(-8), y1));
    a = A::add(a, A::mul(T(16), ymid));
    T b = A::mul(dc.fc[2], f0);
    b = A::add(b, A::mul(dc.fc[3], f1));
    b = A::add(b, A::mul(T(18), y0));
    b = A::add(b, A::mul(T(14), y1));
    b = A::add(b, A::mul(T(-32), ymid));
    T c = A::mul(dc.fc[4], f0);
    c = A::add(c, A::mul(dtk, f1));
    c = A::add(c, A::mul(T(-11), y0));
    c = A::add(c, A::mul(T(-5), y1));
    c = A::add(c, A::mul(T(16), ymid));
    ca = a;
    cb = b;
    cc = c;
    cd = A::mul(dtk, f0);
}

// The fitted quartic of one element at x (x2 = x^2, x3 = x^3, x4 = x^4), interp.py:55-67
template <typename T>
__device__ __forceinline__ T quartic_eval(T ca, T cb, T cc, T cd, T y0, T x, T x2, T x3, T x4) {
    using A = Ar<T>;
    T v = A::mul(ca, x4);
    v = A::add(v, A::mul(cb, x3));
    v = A::add(v, A::mul(cc, x2));
    v = A::add(v, A::mul(cd, x));
    return A::add(v, y0);
}
