// b2ode_fused.cu -- whole adaptive solve in ONE persistent kernel for built-in right-hand sides (DESIGN.md §4.2).
//
// SURVEY.md 8(f)-2.  When `func` is one of the library's own right-hand sides (tfdiffeq_b200/rhs.py), the user
// callable does not have to be called from the host at all: every trajectory of the batch lives in the
// registers of one thread -- state, all s stage derivatives -- for the entire solve; the only HBM traffic is
// the (T, B, D) solution slab, written once.  The reference semantics are kept exactly: ONE step size for
// the whole batch and a tolerance that is a global scalar over the whole tensor (tfdiffeq/misc.py:257), so
// every attempt needs one grid-wide all-reduce (control_allreduce; cooperative launch guarantees co-residency),
// after which every block holds the bit-identical total and evaluates the controller itself.
// The arithmetic is the same as the generic path's kernels (same helpers from b2ode_dev.cuh, same operation
// order: rk_common.py:49-60, misc.py:250-287, interp.py:6-67), only the reduction order differs.

#include "b2ode_dev.cuh"
#include "b2ode_rhs.cuh"
#include "b2ode_bp.cuh"
#include "b2ode_pay16.cuh"
#include <stdlib.h>
#include <mutex>

// ------------------------------------------------------------------------------------------------
// optional timeline stamps (-DB2ODE_FUSED_TRACE, scripts/fused_trace.py): thread 0 of two blocks records clock64() at the
// phase boundaries of attempts [8, 8 + kTraceAttempts); compiled out of the shipped library
// ------------------------------------------------------------------------------------------------
#ifdef B2ODE_FUSED_TRACE
constexpr int kTraceAttempts = 64, kTracePhases = 16;
__device__ unsigned long long g_fused_trace[2 * kTraceAttempts * kTracePhases];
// `dep` is a value that only exists after the event being stamped (a word read after a barrier / received from a poll):
// the clock read is predicated on it, so ptxas cannot hoist the read above the event (an unanchored clock64() was observed
// to float above BAR.SYNC)
#define FTRACE_DEP(att, ph, dep)                                                                                 \
    do {                                                                                                         \
        if ((unsigned)(dep) != 0x7ffffff3u && (threadIdx.x == 0 || threadIdx.x == blockDim.x - 32) /* single-GPU traces: the control warp is the last warp */ &&            \
            (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1) && (att) >= 8 && (att) < 8 + kTraceAttempts)        \
            g_fused_trace[((blockIdx.x == 0 ? 0 : 1) * kTraceAttempts + ((att)-8)) * kTracePhases + (ph)] = clock64(); \
    } while (0)
#define FTRACE(att, ph) FTRACE_DEP(att, ph, 0)
extern "C" int b2ode_debug_fused_trace(unsigned long long *out) {
    B2_CUDA(cudaMemcpyFromSymbol(out, g_fused_trace, sizeof(g_fused_trace)));
    return 0;
}
#else
#define FTRACE(att, ph) do { } while (0)
#define FTRACE_DEP(att, ph, dep) do { } while (0)
#endif

// Block shape: compute warps carrying trajectory warps of 32 consecutive trajectories (one or two per thread, FusedShape),
// one control warp and, in a shared-step group, one comm warp; fused_geometry picks the block size per batch.

// ------------------------------------------------------------------------------------------------
// Grid-wide (and group-wide) all-reduce of two 64-bit values and a flag per attempt, built for LATENCY: measured on the
// round-1 kernel (scripts/fused_trace.py) an attempt cost 15.7k cycles of which only 3.1k were the Runge-Kutta arithmetic;
// the rest was two block reductions with __syncthreads (1.2k + 2.9k), an atomic grid barrier (2.5k), the serial controller
// (3.1k) and the dense output (2.4k), all on every thread's critical path.  Now (DESIGN.md §4.2):
//   * one CONTROL WARP per block owns the exchange; the compute warps hand it their trajectory-warp partials through shared
//     memory and a named barrier (bar.arrive, they do not wait), write the dense output of the step SPECULATIVELY while
//     the control warp talks to the rest of the GPU, and pick the decision up at a second named barrier;
//   * every block stores one 16-byte tagged partial (b2ode_pay16.cuh) and bumps a relaxed arrival counter; every control
//     warp fetches all partials and reduces them in a fixed order (control_allreduce); with a shared-step group every block
//     also stores its partial into every peer's mailbox, where the peers' comm warps gather it (remote_gather);
//   * every control warp then evaluates the (cheap, now low-latency) controller redundantly and bit-identically.
// ------------------------------------------------------------------------------------------------

// The tableau (runtime values) of every kernel family in this file.  Structural zeros are multiplied like any other
// coefficient, as the reference does (misc.py:114-121: its zero test never fires): x + 0 * k == x for finite k, so results
// equal the generic path's.  rtol0 and atol0, the first segment's tolerances, are adjacent because the kernels load them
// as a pair.
struct Tableau {
    double beta[B2ODE_MAXK][B2ODE_MAXK];
    double c_sol[B2ODE_MAXK], c_error[B2ODE_MAXK], c_mid[B2ODE_MAXK];
    int fsal;
    double rtol0, atol0;
};

static void fill_tableau(Tableau &t, const b2ode_adaptive_desc &d) {
    for (int i = 0; i < B2ODE_MAXK; ++i) {
        for (int j = 0; j < B2ODE_MAXK; ++j) t.beta[i][j] = d.beta[i][j];
        t.c_sol[i] = d.c_sol[i];
        t.c_error[i] = d.c_error[i];
        t.c_mid[i] = d.c_mid[i];
    }
    t.fsal = d.fsal;
    t.rtol0 = d.rtol[0];
    t.atol0 = d.atol[0];
}

struct FusedParams {
    b2ode_state *st;
    unsigned long long *part2;   // [2][gridDim.x][2] u64: 16-byte tagged block partials, double buffered by exchange parity
    unsigned *ctr;               // monotonically increasing arrival counter (zeroed by the host before the launch)
    const void *y0;
    void *out;
    // optional streaming of the solution to the host: `progress` counts output rows completed over all blocks, `host_mark`
    // (page-locked host memory, mapped) receives the number of leading rows that are complete on EVERY block, so that the
    // host can issue device-to-host copies behind the solve (b2ode_fused_desc.host_mark)
    unsigned *progress;
    int *host_mark;
    long long n_traj;       // trajectories on this rank
    int ncw;                // trajectory warps (32 consecutive trajectories each) per block; see FusedShape
    int have_first_step;
    double t_start, first_step;
    double time_sign;       // -1 when integrating the reversed system (misc.py:318-321)
    double rhs[8];
    const void *rhs_data;   // device buffer of staged weights (RhsCubicMLP), else null
    Tableau tab;
    CtrlParams c;
    CommParams comm;
};

__device__ __forceinline__ unsigned long long umax64(unsigned long long a, unsigned long long b) { return a > b ? a : b; }

// two 64-bit lanes of payload + one flag bit.  MODE 0: (a: sum >= 0, b: bit pattern of a non-negative double, combined
// with an unsigned max -- NaN patterns sort above +inf, so it is a NaN-propagating max for free); MODE 1: (a, b: sums)
template <int MODE>
__device__ __forceinline__ Pay pay_identity() {
    Pay r;
    r.a = 0.0;
    r.b = 0ull;       // +0.0 as a double, 0 as a max identity
    r.flag = 0u;
    return r;
}

template <int MODE>
__device__ __forceinline__ Pay pay_combine(const Pay &x, const Pay &y) {
    Pay r;
    r.a = x.a + y.a;
    if (MODE == 0) r.b = x.b > y.b ? x.b : y.b;
    else r.b = (unsigned long long)__double_as_longlong(__longlong_as_double((long long)x.b) + __longlong_as_double((long long)y.b));
    r.flag = x.flag | y.flag;
    return r;
}

template <int MODE>
__device__ __forceinline__ Pay pay_warp_reduce(Pay x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Pay y;
        y.a = __shfl_xor_sync(0xffffffffu, x.a, o);
        y.b = __shfl_xor_sync(0xffffffffu, x.b, o);
        y.flag = __shfl_xor_sync(0xffffffffu, x.flag, o);
        x = pay_combine<MODE>(x, y);
    }
    return x;       // every lane holds the warp total (a + b == b + a bitwise, so all lanes agree)
}

__device__ __forceinline__ void named_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void named_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// blockDim.x, read afresh at every use (volatile: not merged with other reads).  A barrier count computed once and kept across
// the compute warps' attempt loop is spilled there by ptxas and reloaded from local memory in front of every barrier.
__device__ __forceinline__ int ntid_fresh() {
    int v;
    asm volatile("mov.u32 %0, %%ntid.x;" : "=r"(v));
    return v;
}

// -x when `neg`, else x: exact (a sign-bit flip), and one integer instruction instead of an FP64 negation and two selects
__device__ __forceinline__ double negate_if(double x, bool neg) {
    return __longlong_as_double(__double_as_longlong(x) ^ (neg ? (long long)0x8000000000000000ull : 0ll));
}
__device__ __forceinline__ float negate_if(float x, bool neg) { return __int_as_float(__float_as_int(x) ^ (neg ? (int)0x80000000u : 0)); }

// The polls below use WEAK loads (ld.global.cg: they overlap; strong loads of one warp do not), and to the PTX memory
// model a weak load of an unchanged address may be assumed to return the same value again: ptxas is entitled to hoist such
// a load out of a polling loop, or to drop the loop ("it must terminate, so its condition holds") -- and does, once the loop
// is simple enough.  Every polling round therefore offsets its addresses by this value, which is always 0 but which ptxas
// cannot know: the loads are loop-variant and have to be issued again.
__device__ __forceinline__ unsigned long long opaque_zero() {
    unsigned long long c;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(c));
    return c >> 63;
}

constexpr int kGatherPerLane = 5;        // 160 blocks gathered with every poll in flight (H100: 132 SMs x 1 block)
constexpr int kGatherRanks = 3;          // source ranks remote_gather polls per round (15 weak loads per lane)

// shared scratch of one block
struct FusedShared {
    Pay part[32];                  // trajectory-warp partials (one per control-warp lane)
    unsigned long long rlane[B2ODE_MAXPEERS][32][2];   // per-lane sums of the OTHER ranks' partials (comm warp -> control warp)
    Pay tot;                       // totals of the initial-step reductions (read by every thread)
    struct {
        double dt_next;
        int accept, done;
        unsigned status;
    } ctl;                         // what the control warp hands to the compute warps
};

constexpr int kBarPartials = 1, kBarDecision = 2, kBarRows = 3, kBarRowsReady = 4, kBarRemote = 5, kBarFirstStep = 6;

// The quartic fit's constants of one attempt (DenseConst, b2ode_dev.cuh) from the tableau; `dtc` carries the sign of the time
// direction (see `rhs` in k_fused_adaptive).
template <typename T, int S>
__device__ __forceinline__ DenseConst<T, S> dense_const(const Tableau &tab, T dtc) {
    DenseConst<T, S> dc;
#pragma unroll
    for (int j = 0; j < S; ++j) dc.cmid[j] = Ar<T>::mul(dtc, (T)tab.c_mid[j]);
#pragma unroll
    for (int q = 0; q < 5; ++q) dc.fc[q] = Ar<T>::mul(fit_coef<T>(q), dtc);
    return dc;
}

// acc[u][d] = sum_{j < J} coef(j) * k(j, u, d) for U rows of D elements (rk_common.py:49-60, misc.py:121): the stage input,
// solution, error and midpoint combines of k_fused_adaptive and k_rows_adaptive.  The first product is not added to a zero
// (that would turn -0 into +0); j runs outermost, then the row, then the element, and coef(j) is formed once per j.
template <typename T, int U, int D, typename C, typename K>
__device__ __forceinline__ void tableau_combine(T (&acc)[U][D], int J, C &&coef, K &&k) {
#pragma unroll
    for (int j = 0; j < J; ++j) {
        const T c = coef(j);
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
            for (int d = 0; d < D; ++d) {
                const T term = Ar<T>::mul(c, k(j, u, d));
                acc[u][d] = (j == 0) ? term : Ar<T>::add(acc[u][d], term);
            }
    }
}

// One row's terms of the error norm (misc.py:256-263), in element order: sum err^2 in fp64, max(|y0|, |y1|) as the bit
// pattern of a non-negative double (compared as an integer: NaN patterns sort above +inf, so the max propagates NaN), and
// whether y0 holds an inf or NaN (dopri5.py:100).
struct NormTerms {
    double ssq;
    unsigned long long amax;
    bool bad0;
};

template <typename T, int D>
__device__ __forceinline__ NormTerms norm_terms(const T (&err)[D], const T (&y0)[D], const T (&y1)[D]) {
    double sum = 0.0;
    unsigned long long m0 = 0ull, m1 = 0ull;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        const double ed = (double)err[d];
        sum += ed * ed;
        m0 = umax64(m0, (unsigned long long)__double_as_longlong(fabs((double)y0[d])));
        m1 = umax64(m1, (unsigned long long)__double_as_longlong(fabs((double)y1[d])));
    }
    NormTerms r;
    r.ssq = sum;
    r.amax = umax64(m0, m1);
    r.bad0 = m0 >= 0x7ff0000000000000ull;
    return r;
}

// _select_initial_step on one row (misc.py:183-226): scale = atol + |y0| rtol, and s0 = sum (y0 / scale)^2,
// s1 = sum (f0 / scale)^2 in fp64.  A row that is not `live` (a lane past the batch) still forms its scale but adds nothing.
template <typename T, int D>
__device__ __forceinline__ void init_sums(const T (&y)[D], const T (&f0)[D], T rtol, T atol, T (&scale)[D], double &s0,
                                          double &s1, bool live = true) {
    using A = Ar<T>;
    s0 = 0.0;
    s1 = 0.0;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        scale[d] = A::add(atol, A::mul(A::abs(y[d]), rtol));
        if (live) {
            const double q0 = (double)A::div(y[d], scale[d]), q1 = (double)A::div(f0[d], scale[d]);
            s0 += q0 * q0;
            s1 += q1 * q1;
        }
    }
}

// misc.py:238-240 on one row: sum ((f1 - f0) / scale)^2 in fp64, f1 the derivative at the probe y0 + h0 f0
template <typename T, int D>
__device__ __forceinline__ double init_s2(const T (&f1)[D], const T (&f0)[D], const T (&scale)[D]) {
    double s2 = 0.0;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        const double q = (double)Ar<T>::div(Ar<T>::sub(f1[d], f0[d]), scale[d]);
        s2 += q * q;
    }
    return s2;
}

// What the control warp hands to the compute warps for the speculative dense output of an attempt (written before its
// arrival on kBarRows, read after the compute warps' kBarRows): the fit coefficients and, for each of the first rows of
// the step, x = (t_out - t0) / (t1 - t0) and its powers x^2, x^3, x^4.
template <typename T, int S>
struct DenseShared {
    DenseConst<T, S> k;
    T x[3][4];
};

// The products of an attempt's step with the tableau, the same for every trajectory: dt·beta[s][j] (j <= s < S - 1),
// dt·c_error[j] and dt·c_sol[j], each with the sign of the time direction (see `rhs` in k_fused_adaptive).  The control warp
// forms them, one per lane, as soon as it knows the step, and publishes them here before its kBarDecision arrival; the compute
// warps read them as broadcasts in the stages and the error estimate of the attempt.  Rewritten only after the next
// kBarPartials, when every compute warp has read them.
template <typename T, int S>
struct StageConst {
    static constexpr int nb = S * (S - 1) / 2, n = nb + 2 * S;
    static constexpr __host__ __device__ int beta(int s, int j) { return s * (s + 1) / 2 + j; }
    static constexpr __host__ __device__ int err(int j) { return nb + j; }
    static constexpr __host__ __device__ int sol(int j) { return nb + S + j; }
    __align__(16) T c[n];
};

// tableau coefficient behind StageConst<T, S>::c[idx]
template <typename T, int S>
__device__ __forceinline__ T stage_coef(const FusedParams &p, int idx) {
    using SC = StageConst<T, S>;
    if (idx >= SC::sol(0)) return (T)p.tab.c_sol[idx - SC::sol(0)];
    if (idx >= SC::err(0)) return (T)p.tab.c_error[idx - SC::err(0)];
    int s = 0;
    while (idx > s) idx -= ++s;          // row s of beta holds s + 1 coefficients
    return (T)p.tab.beta[s][idx];
}

// Called by the COMM warp (blocks of a shared-step group have one: a second service warp without trajectories): fetch the
// partials every peer wrote into this rank's mailbox over NVLink and leave, per source rank, each LANE's share (blocks
// lane, lane + 32, ... summed in that order) in shared memory; the control warp folds the ranks in rank order and does the
// one butterfly.  The comm warp starts polling the moment an exchange begins, so the peers' data is fetched while the
// control warp is still in the intra-GPU phase: the NVLink hop (~2070 cycles) hides behind it.  kGatherRanks source ranks
// are polled together, round by round, until every partial carries the tag of `seq`.
template <int MODE>
__device__ __forceinline__ void remote_gather(const FusedParams &p, FusedShared &sh, unsigned seq) {
    const int nranks = p.comm.nranks, lane = threadIdx.x & 31, rank = p.comm.rank;
    constexpr int RG = kGatherRanks;                        // source ranks per batch
    constexpr int NL = RG * kGatherPerLane;                 // loads in flight per lane
    const unsigned long long *base = &p.comm.box[rank]->fused_part[seq & 1u][0][0][0] + (size_t)lane * 2;
    const unsigned tag = pay_tag(seq);
    for (int i0 = 0; i0 < nranks - 1; i0 += RG) {
        // The poll loop is INSTRUCTION bound (one warp, every load followed by its validation), so it is kept minimal: one
        // pointer per source rank, loads at immediate offsets and without predicates -- a slot past the source's grid, or
        // of a rank past the group, is just memory of the mailbox (fused_part has kMaxFusedBlocks >= 32 * kGatherPerLane
        // slots per rank) whose content is ignored -- and a two-instruction tag test per load.  Slots that were valid a
        // round ago stay valid (a buffer is rewritten two exchanges later), so every round simply reloads everything.
        unsigned long long g0[NL], g1[NL];
        const unsigned long long *ptr[RG];
        unsigned mine = 0u;
#pragma unroll
        for (int r = 0; r < RG; ++r) {
            const int i = i0 + r;
            const bool ok = i < nranks - 1;
            const int src = ok ? (i < rank ? i : i + 1) : rank;
            const int G = ok ? p.comm.grid_of[src] : 0;
            ptr[r] = base + (size_t)src * (kMaxFusedBlocks * 2);
            asm volatile("" : "+l"(ptr[r]));                 // (keep it in a register: do not recompute it per load)
#pragma unroll
            for (int q = 0; q < kGatherPerLane; ++q)
                if (lane + 32 * q < G) mine |= 1u << (r * kGatherPerLane + q);
        }
        unsigned got;
        do {
            const unsigned long long z = opaque_zero();
#pragma unroll
            for (int r = 0; r < RG; ++r)
#pragma unroll
                for (int q = 0; q < kGatherPerLane; ++q)
                    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];"
                                 : "=l"(g0[r * kGatherPerLane + q]), "=l"(g1[r * kGatherPerLane + q])
                                 : "l"(ptr[r] + z + 64 * q)
                                 : "memory");
            got = 0u;
#pragma unroll
            for (int k = 0; k < NL; ++k) {
                got |= (pay_mismatch(g0[k], g1[k], tag) == 0u) ? (1u << k) : 0u;
            }
        } while ((got & mine) != mine);
#pragma unroll
        for (int r = 0; r < RG; ++r) {
            const int i = i0 + r;
            if (i >= nranks - 1) continue;
            const int src = i < rank ? i : i + 1;
            Pay acc = pay_identity<MODE>();
#pragma unroll
            for (int q = 0; q < kGatherPerLane; ++q)
                if ((mine >> (r * kGatherPerLane + q)) & 1u)
                    acc = pay_combine<MODE>(acc, pay_unpack16(g0[r * kGatherPerLane + q], g1[r * kGatherPerLane + q]));   // fixed order
            const int G = p.comm.grid_of[src];
            for (int b = lane + 32 * kGatherPerLane; b < G; b += 32) {       // grids beyond 32 * kGatherPerLane blocks
                const unsigned long long *sl = base + (size_t)src * (kMaxFusedBlocks * 2) + (size_t)(b - lane) * 2;
                unsigned long long a0, a1;
                do {
                    asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(a0), "=l"(a1) : "l"(sl + opaque_zero()) : "memory");
                } while (!pay_valid16(a0, a1, seq));
                acc = pay_combine<MODE>(acc, pay_unpack16(a0, a1));
            }
            unsigned long long ab = (unsigned long long)__double_as_longlong(acc.a);
            if (acc.a != acc.a) ab = 0x7ff8000000000000ull;
            sh.rlane[src][lane][0] = (ab & 0x7fffffffffffffffull) | ((unsigned long long)(acc.flag & 1u) << 63);
            sh.rlane[src][lane][1] = acc.b;
        }
    }
    asm volatile("bar.arrive %0, %1;" ::"r"(kBarRemote), "r"(64) : "memory");
}

// Called by the CONTROL warp (all 32 lanes, convergent) once the compute warps' partials are in sh.part[0 .. ncw).
// `epoch` counts the exchanges of this launch (1, 2, ...).  Returns the group-wide totals in every lane of every block of
// every rank, bit-identical everywhere.
//
// Why the exchange is built this way (costs from microbenchmarks of the protocol, scripts/micro/grid_barrier.cu and
// nvlink_pingpong.cu, on the previous target; not re-measured on H100):
//   * a gpu- or sys-scope STRONG load (ld.relaxed / acquire / volatile, atomic read) costs 500-700 cycles and the strong loads
//     of one warp do not overlap: a flag protocol that polls k words pays k round trips per poll; a leader gathering 147
//     messages with 5 polls per lane pays ~10 serialised round trips (7.3k cycles per all-reduce; two-level 13.4k);
//   * one atomic arrival counter + one polled word: 1.9k; weak ld.global.cg loads always read the L2 and pipeline;
//   * a fence (red.release) in front of the arrival costs a MEMBAR.GPU = the store's round trip;
//   * one NVLink hop (remote write -> visible to a poll of local memory) is ~2070 cycles whatever the instructions, +520 per
//     extra polled word; REMOTE atomics on one address serialise badly (147 blocks x 7 peers bumping per-source counters:
//     11.5 us per attempt at 8 GPUs against 4.2 us on one); an intra-GPU all-reduce followed by one message per peer puts
//     the hop behind the whole local phase (+3.1 us per attempt at 2 GPUs).
// Hence: every block stores its 16-byte tagged partial LOCALLY and, over NVLink, into EVERY peer's mailbox (plain stores: the
// tag validates the data, no flag, no remote atomic).  Inside the GPU one RELAXED arrival atomic orders nothing (no fence: a
// reader that finds a stale tag re-reads), lane 0 spins on the counter with one strong load per poll, then all partials
// are fetched with weak loads that overlap.  The peers' partials, which travel during the local phase, are gathered by a
// dedicated COMM warp (remote_gather) and handed to the control warp through shared memory; ranks combine in rank order.
template <int MODE>
__device__ __forceinline__ Pay control_allreduce(const FusedParams &p, FusedShared &sh, int ncw, unsigned epoch, unsigned seq0,
                                                 unsigned long long hw2 = 0ull /* Mailbox::fused_hw[0..1] at kernel start */,
                                                 int att = -1) {
    const int lane = threadIdx.x & 31;
    Pay x = (lane < ncw) ? sh.part[lane] : pay_identity<MODE>();
    x = pay_warp_reduce<MODE>(x);                                         // block total, all lanes
    FTRACE_DEP(att, 2, __double_as_longlong(x.a));
    const int nranks = p.comm.nranks > 1 ? p.comm.nranks : 1, rank = p.comm.rank;
    const int G = (int)gridDim.x;
    // buffer parity follows the PERSISTENT sequence number, so the alternation continues across launches: a rank that has
    // already started the next solve cannot overwrite a partial a slower rank has not read yet
    const unsigned seq = seq0 + epoch, par = seq & 1u;
    unsigned long long w0, w1;
    pay_pack16(x, seq, w0, w1);
    if (nranks > 1 && epoch <= 2u && lane < nranks && lane != rank) {
        // first use of this buffer in this solve: slots the previous writer of the buffer filled and this (smaller) grid does
        // not are poisoned in every peer's mailbox, so that no later solve can take them for fresh partials
        const int hw = (int)(par ? (unsigned)(hw2 >> 32) : (unsigned)hw2);
        for (int b = G + (int)blockIdx.x; b < hw && b < kMaxFusedBlocks; b += G) {
            unsigned long long *dst = &p.comm.box[lane]->fused_part[par][rank][b][0];
            asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(kPoisonW0), "l"(kPoisonW1) : "memory");
        }
    }
    if (nranks > 1 && lane < nranks && lane != rank) {                    // lane q: this block's partial -> rank q, over NVLink
        unsigned long long *dst = &p.comm.box[lane]->fused_part[par][rank][blockIdx.x][0];
        asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(w0), "l"(w1) : "memory");
    }
    if (G > 1) {
        unsigned long long *slots = p.part2 + (size_t)par * G * 2;
        if (lane == 0) {
            asm volatile("st.relaxed.gpu.global.v2.u64 [%0], {%1, %2};" ::"l"(slots + (size_t)blockIdx.x * 2), "l"(w0), "l"(w1) : "memory");
            asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(p.ctr) : "memory");
            const unsigned target = epoch * (unsigned)G;
            unsigned v;
            do {
                asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p.ctr) : "memory");
            } while ((int)(v - target) < 0);
        }
        __syncwarp();
        FTRACE(att, 3);
        // this LANE's share of this GPU's partials (blocks lane, lane + 32, ...: fixed order).  All arrivals have been seen, so
        // the partials are almost always there: five unconditional weak loads in flight (a lane without a block at
        // lane + 32 q reads slot 0 and ignores it), then the tag test; a stale tag -- the relaxed arrival overtook its
        // data -- is re-read with strong loads, which the compiler may not hoist or elide.
        unsigned long long g0[kGatherPerLane], g1[kGatherPerLane];
#pragma unroll
        for (int q = 0; q < kGatherPerLane; ++q) {
            const int b = lane + 32 * q;
            asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(g0[q]), "=l"(g1[q]) : "l"(slots + (size_t)(b < G ? b : 0) * 2) : "memory");
        }
        x = pay_identity<MODE>();
#pragma unroll
        for (int q = 0; q < kGatherPerLane; ++q) {
            const int b = lane + 32 * q;
            if (b < G) {
                while (!pay_valid16(g0[q], g1[q], seq))
                    asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(g0[q]), "=l"(g1[q]) : "l"(slots + (size_t)b * 2) : "memory");
                x = pay_combine<MODE>(x, pay_unpack16(g0[q], g1[q]));
            }
        }
        for (int b = lane + 32 * kGatherPerLane; b < G; b += 32) {         // grids beyond 32 * kGatherPerLane blocks
            unsigned long long a0, a1;
            do {
                asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(a0), "=l"(a1) : "l"(slots + (size_t)b * 2) : "memory");
            } while (!pay_valid16(a0, a1, seq));
            x = pay_combine<MODE>(x, pay_unpack16(a0, a1));
        }
    } else {
        x = (lane == 0) ? pay_unpack16(w0, w1) : pay_identity<MODE>();   // (the transported form, like everybody else's)
    }
    if (nranks == 1) return pay_warp_reduce<MODE>(x);
    asm volatile("bar.sync %0, %1;" ::"r"(kBarRemote), "r"(64) : "memory");                    // the comm warp has the peers' lane sums
    Pay tot = pay_identity<MODE>();
    for (int q = 0; q < nranks; ++q) {                                     // rank order, per lane: identical on every GPU
        Pay v = x;
        if (q != rank) {
            const unsigned long long a = sh.rlane[q][lane][0];
            v.flag = (unsigned)(a >> 63);
            v.a = __longlong_as_double((long long)(a & 0x7fffffffffffffffull));
            v.b = sh.rlane[q][lane][1];
        }
        tot = (q == 0) ? v : pay_combine<MODE>(tot, v);
    }
    return pay_warp_reduce<MODE>(tot);                                     // one butterfly for the whole group
}

// The controller of the persistent kernel (one segment, the reference's controller: misc.py:250-287), written for the
// shortest dependent chain -- it sits on the critical path of every attempt with the whole GPU waiting:
//   accept  <=>  mean((err/tol)^2) <= 1  <=>  sum err^2 <= tol^2 * n         (no division; fp32 states compare in fp32,
//                                                                             i.e. against the largest double that rounds to 1.0f)
//   dt_next = dt / clamp(sqrt(m)^e / safety, 1/ifactor, 1/dfactor) = dt * clamp(safety * 2^(-e/2 * log2 m), dfactor', ifactor)
//   with log2 m = log2(sum err^2) - log2(tol^2 n): two independent logarithms, one exp2, no division, no sqrt.
// The reference rounds m to the state dtype before both of its tests (accept: m <= 1; keep dfactor: m >= 1).  An fp32 m
// rounds to 1.0f exactly when the unrounded ratio lies in [1 - 2^-25, 1 + 2^-24], so fp32 states compare sum err^2 with
// tol^2 n scaled by those two ends (one multiply each, off the logarithms' chain).  The products are rounded in fp64,
// which leaves a band of about 2^-53 relative at each end where the two tests may disagree.
// dt_next's relative error against a correctly rounded evaluation of the reference's formula at the same m is bounded in
// tests/controller_cases.py (dt_bound): (e/2) ln2 2^-52 (|log2 sum err^2| + |log2 tol^2 n|) from the two logarithms (1 ulp
// each), whose difference cancels, plus a few 2^-53 from exp2 (2 ulp), the multiplies and the ratio's own error; an fp32
// state adds up to 1.5 e 2^-24, because m and sqrt(m) are not rounded to fp32 here.  The clamps multiply by ifactor and
// dfactor where the reference divides by their fp64 reciprocals (2 2^-53).  dt is a free parameter of the method; the
// parity bars are on the solution (1e-6 / 1e-3).
// Called by all 32 lanes of the control warp, convergent (it shuffles).
template <typename T>
__device__ __forceinline__ CtrlDecision ctrl_fast(const CtrlParams &c, double ssq, double mm, bool bad0, double dt) {
    constexpr bool f32 = std::is_same<T, float>::value;
    const T tol = Ar<T>::add((T)c.atol[0], Ar<T>::mul((T)c.rtol[0], (T)mm));
    const double tol2n = (double)tol * (double)tol * (double)c.n_global[0];
    const double bound = f32 ? tol2n * (1.0 + 5.9604644775390625e-08) : tol2n;    // (T)m <= 1
    const double below = f32 ? tol2n * (1.0 - 2.98023223876953125e-08) : tol2n;   // (T)m < 1
    CtrlDecision d;
    d.bad0 = bad0;
    d.accept = ssq <= bound;
    {
        // the two logarithms are independent: lane 0 takes log2(ssq), the other lanes log2(tol2n) (one log2 on the chain)
        const double lg = log2(((threadIdx.x & 31) == 0) ? ssq : tol2n);
        const double L = __shfl_sync(0xffffffffu, lg, 0) - __shfl_sync(0xffffffffu, lg, 1);
        const double df = (ssq < below) ? 1.0 : c.dfactor;
        const double rf = c.safety * exp2(-0.5 * c.exponent * L);
        d.dt_next = (ssq == 0.0) ? dt * c.ifactor : dt * nan_min(c.ifactor, nan_max(df, rf));
    }
    d.m = 0.0;       // filled in off the critical path
    return d;
}

// ------------------------------------------------------------------------------------------------
// the persistent solve.  Block = compute warps (TPT trajectories per thread) + 1 control warp + (with a shared-step group)
// 1 comm warp.  The block's p.ncw * 32 trajectories form p.ncw TRAJECTORY WARPS of 32 consecutive trajectories; compute
// warp w carries trajectory warps w, w + pcw, ... (pcw compute warps).  A trajectory warp has its own butterfly, partial
// slot and place in s_rows, so the partition of the batch and the order of every reduction are those of one trajectory
// per thread: the results do not depend on TPT.  Two trajectories per thread halve the warps that hold a block's batch and
// so raise the register budget of a thread; the two trajectories' stages are independent chains, interleaved.
//
// MAXT is the block's trajectory budget, stated as the threads it would take at one trajectory per thread: at most
// MAXT / 32 - 1 trajectory warps (one service warp; one fewer with a shared-step group).  The block itself has
// FusedShape<T, RHS, S, MAXT>::threads threads at most.  (With TPT = 2 the launch bound asks for one block per SM: without it
// ptxas caps some instances at 96 registers and spills.)
// ------------------------------------------------------------------------------------------------

// compute warps + service warps of a block of `ntw` trajectory warps at `tpt` trajectories per thread
constexpr int fused_warps(int ntw, int tpt, int nsvc) { return (ntw + tpt - 1) / tpt + nsvc; }
constexpr int cmax(int a, int b) { return a > b ? a : b; }

// Trajectories per thread of an instantiation: two for the 7-k tableaus (dopri5), where that lifts the register cap from
// 96 (18 warps per block) to 168 (10 warps); fp64 Kepler (D = 4) spills more with two than with one and keeps one.  The
// 2-, 4- and 14-k tableaus have room at one (<= 128 and <= 255 registers) and would spill with two.
template <typename T, typename RHS, int S, int MAXT>
struct FusedShape {
    static constexpr int tpt = (S == 7 && !(std::is_same<T, double>::value && RHS::D > 3)) ? 2 : 1;
    // threads of the largest block: alone MAXT / 32 - 1 trajectory warps + 1 service warp, in a group MAXT / 32 - 2 + 2
    static constexpr int threads = 32 * cmax(fused_warps(MAXT / 32 - 1, tpt, 1), fused_warps(MAXT / 32 - 2, tpt, 2));
    static constexpr int min_blocks = tpt > 1 ? 1 : 0;
};

template <typename T, typename RHS, int S, int MAXT>
__global__ void __launch_bounds__(FusedShape<T, RHS, S, MAXT>::threads, FusedShape<T, RHS, S, MAXT>::min_blocks)
k_fused_adaptive(const __grid_constant__ FusedParams p) {
    constexpr int TPT = FusedShape<T, RHS, S, MAXT>::tpt;
    using A = Ar<T>;
    constexpr int D = RHS::D;
    constexpr int kMaxTraj = MAXT - 32;                  // trajectories of the largest block (one service warp)
    __shared__ FusedShared sh;
    __shared__ T sw[RHS::kSmem];
    __shared__ DenseShared<T, S> sdc;
    __shared__ StageConst<T, S> ssc;
    constexpr int kDenseRows = (3 * kMaxTraj * D * (int)sizeof(T) + (int)sizeof(FusedShared) + RHS::kSmem * (int)sizeof(T) +
                                (int)sizeof(DenseShared<T, S>) + (int)sizeof(StageConst<T, S>) + 256 <= 48 * 1024) ? 3 : 2;
    __shared__ __align__(16) T s_rows[kDenseRows][kMaxTraj * D];     // dense-output rows of the step, waiting for the decision
    const int nthreads = blockDim.x;
    const bool grouped = p.comm.nranks > 1;
    const int nsvc = grouped ? 2 : 1;                    // service warps: control (+ comm with a shared-step group)
    const int pcw = (nthreads >> 5) - nsvc;              // compute warps
    const int ncw = p.ncw;                               // trajectory warps: pcw * TPT - ncw < TPT
    const int nloc = 32 * (pcw + 1);                     // compute warps + control warp (barriers the comm warp is not part of)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool is_control = warp == pcw;
    // persistent exchange number of the cross-GPU receive area (it survives across solves in the mailbox)
    const unsigned ll_base = grouped ? (unsigned)p.comm.box[p.comm.rank]->ll_seq : 0u;
    const unsigned long long hw2 = (grouped && is_control) ? *(const volatile unsigned long long *)p.comm.box[p.comm.rank]->fused_hw : 0ull;
    stage_weights<T, RHS>(p.rhs, p.rhs_data, sw, nthreads);
    const int n_out = p.c.n_out;
    const double *__restrict__ t_out = p.c.t_out;

    if (is_control) {
        // ================================ control warp =================================================
        unsigned epoch = 0;
        double t_cur = p.t_start, dt;
        unsigned status = 0;
        if (p.have_first_step) {
            dt = p.first_step;
        } else {
            // misc.py:226-247 with the two reductions of _select_initial_step
            named_sync(kBarPartials, nloc);
            Pay r = control_allreduce<1>(p, sh, ncw, ++epoch, ll_base, hw2);
            if (lane == 0) sh.tot = r;
            named_arrive(kBarDecision, nthreads);
            Partial tot;
            tot.v[0] = r.a;
            tot.v[1] = __longlong_as_double((long long)r.b);
            tot.v[2] = tot.v[3] = 0.0;
            T d1max;
            const T h0 = init_h0<T>(p.c, &tot, 1, &d1max);
            named_sync(kBarPartials, nloc);
            r = control_allreduce<1>(p, sh, ncw, ++epoch, ll_base, hw2);
            if (lane == 0) sh.tot = r;
            named_arrive(kBarDecision, nthreads);
            tot.v[0] = r.a;
            dt = (double)init_dt<T>(p.c, &tot, 1, h0, d1max);
        }
        // the stage constants of the coming attempt (StageConst): this lane's tableau coefficients, loop invariant, times the
        // signed step; the compute warps pick the first attempt's up at kBarFirstStep, every later one's at kBarDecision
        constexpr int kSc = StageConst<T, S>::n, kScLane = (kSc + 31) / 32;
        T scoef[kScLane];
#pragma unroll
        for (int q = 0; q < kScLane; ++q) scoef[q] = (lane + 32 * q < kSc) ? stage_coef<T, S>(p, lane + 32 * q) : T(0);
        const bool rev = (T)p.time_sign < T(0);
        auto publish_stage = [&](double dtn) {
            const T dtk = negate_if((T)dtn, rev);
#pragma unroll
            for (int q = 0; q < kScLane; ++q)
                if (lane + 32 * q < kSc) ssc.c[lane + 32 * q] = A::mul(dtk, scoef[q]);
        };
        publish_stage(dt);
        named_arrive(kBarFirstStep, nloc);
        int cur = 1;
        int done = (n_out <= 1) ? 1 : 0;
        if (!done && step_underflows(t_cur, dt)) {
            status |= B2ODE_ST_UNDERFLOW;
            done = 1;
        }
        // bookkeeping for the final state
        int late_rows = 0;     // host streaming: rows of a long step whose completion is accounted one barrier later
        double m_last = 0.0, t_prev = t_cur, dt_last = 0.0;
        unsigned long long n_acc = 0, n_rej = 0;
        long long nadv = 0;
        int att = 0;
        while (!done) {
            FTRACE(att, 0);
            // everything that does not depend on the reduction, computed while the compute warps work
            const double t1_acc = t_cur + dt;
            const int c2 = next_cursor(t_out, cur, n_out, t1_acc);
            if (c2 > cur) {
                // the attempt's dense-output constants, in the operations and order of the compute warps' fit / eval_row
                // (the compute warps of the previous attempt are done reading sdc: they arrived on kBarRowsReady)
                const T dtk = negate_if((T)dt, rev), t0s = (T)t_cur, den = A::sub((T)t1_acc, t0s);
                if (lane < S) sdc.k.cmid[lane] = A::mul(dtk, (T)p.tab.c_mid[lane]);
                if (lane < 5) sdc.k.fc[lane] = A::mul(fit_coef<T>(lane), dtk);
                if (lane < kDenseRows && cur + lane < c2) {
                    const T x = A::div(A::sub((T)__ldg(t_out + cur + lane), t0s), den);
                    const T x2 = A::mul(x, x), x3 = A::mul(x2, x), x4 = A::mul(x3, x);
                    sdc.x[lane][0] = x;
                    sdc.x[lane][1] = x2;
                    sdc.x[lane][2] = x3;
                    sdc.x[lane][3] = x4;
                }
                named_arrive(kBarRows, nloc);                              // the previous step's rows have been copied out
            }
            named_sync(kBarPartials, nloc);                                // the compute warps' partials are in
            if (late_rows) {
                // a long step's extra rows were stored by the compute warps themselves, before this barrier
                __threadfence();
                if (lane == 0) {
                    const unsigned old = atomicAdd(p.progress, (unsigned)late_rows);
                    if (old + (unsigned)late_rows == (unsigned)(cur - 1) * gridDim.x) {
                        __threadfence_system();
                        *(volatile int *)p.host_mark = cur;
                    }
                }
                late_rows = 0;
            }
            FTRACE_DEP(att, 1, sh.part[0].flag);
            const Pay r = control_allreduce<0>(p, sh, ncw, ++epoch, ll_base, hw2, att);
            FTRACE_DEP(att, 4, __double_as_longlong(r.a));
            Partial tot;
            tot.v[0] = r.a;
            tot.v[1] = tot.v[2] = __longlong_as_double((long long)r.b);        // max(max|y0|, max|y1|)
            tot.v[3] = r.flag ? 1.0 : 0.0;                                      // inf or NaN somewhere in y0
            CtrlDecision dec = ctrl_fast<T>(p.c, tot.v[0], tot.v[1], r.flag != 0u, dt);
            const StepAdvance nx = advance_step(dec, status, cur, c2, n_out, nadv, p.c.max_num_steps, t_cur, dt);
            publish_stage(dec.dt_next);
            if (lane == 0) {
                sh.ctl.dt_next = dec.dt_next;
                sh.ctl.accept = dec.accept ? 1 : 0;
                sh.ctl.done = nx.done ? 1 : 0;
                sh.ctl.status = nx.status;
            }
            named_arrive(kBarDecision, nthreads);
            FTRACE_DEP(att, 5, __double_as_longlong(dec.dt_next));
            if (c2 > cur) named_sync(kBarRowsReady, nloc);                  // the compute warps' rows are in shared memory
            if (nx.adv && c2 > cur) {
                // The accepted step's dense-output rows wait in shared memory (written by the compute warps before the
                // decision barrier): this otherwise idle warp streams them to the solution slab with 16-byte stores while
                // the compute warps are already in the next attempt's stages.  The block's part of an output row is one
                // contiguous run of nblk * D elements.
                const long long first = (long long)blockIdx.x * (ncw * 32);
                long long nblk = p.n_traj - first;
                if (nblk > ncw * 32) nblk = ncw * 32;
                const int nel = (int)(nblk > 0 ? nblk * D : 0);
                const long long Nrow = p.n_traj * D;
                const int nrows = (c2 - cur) < kDenseRows ? (c2 - cur) : kDenseRows;
                for (int q = 0; q < nrows; ++q) {
                    T *row = (T *)p.out + (long long)(cur + q) * Nrow + first * D;
                    const T *src = s_rows[q];
                    constexpr int V = 16 / sizeof(T);
                    if ((reinterpret_cast<uintptr_t>(row) & 15u) == 0) {
                        const int nv = nel / V;
                        for (int e = lane; e < nv; e += 32)
                            reinterpret_cast<int4 *>(row)[e] = reinterpret_cast<const int4 *>(src)[e];
                        for (int e = nv * V + lane; e < nel; e += 32) row[e] = src[e];
                    } else {
                        for (int e = lane; e < nel; e += 32) row[e] = src[e];
                    }
                }
                if (p.host_mark) {
                    if (c2 - cur > kDenseRows) {
                        late_rows = c2 - cur;                       // compute warps are still writing rows: account later
                    } else {
                        __threadfence();                            // my rows are visible device-wide before the count moves
                        if (lane == 0) {
                            const unsigned old = atomicAdd(p.progress, (unsigned)(c2 - cur));
                            // rows 1 .. c2-1 complete on every block  <=>  the count reached (c2 - 1) * blocks
                            if (old + (unsigned)(c2 - cur) == (unsigned)(c2 - 1) * gridDim.x) {
                                __threadfence_system();
                                *(volatile int *)p.host_mark = c2;
                            }
                        }
                    }
                }
            }
            {   // the reported error ratio (b2ode_state.msr_max), off the critical path
                const T tol = Ar<T>::add((T)p.c.atol[0], Ar<T>::mul((T)p.c.rtol[0], (T)tot.v[1]));
                dec.m = (double)(T)(tot.v[0] / ((double)tol * (double)tol * (double)p.c.n_global[0]));
            }
            m_last = dec.m;
            dt_last = dt;
            if (dec.accept) {
                n_acc += 1;
                t_prev = t_cur;
                t_cur = nx.t1;
            } else {
                n_rej += 1;
            }
            cur = nx.cur;
            nadv = nx.nadv;
            dt = dec.dt_next;
            status = nx.status;
            done = nx.done;
            ++att;
        }
        if (blockIdx.x == 0 && lane == 0) {
            b2ode_state z;
            memset(&z, 0, sizeof(z));
            z.t0 = t_prev;
            z.t1 = t_cur;
            z.dt = dt;
            z.dt_last = dt_last;
            z.msr_max = m_last;
            z.n_acc = n_acc;
            z.n_rej = n_rej;
            z.attempt = n_acc + n_rej;
            z.n_steps_adv = nadv;
            z.done = 1;
            z.status = status;
            z.cursor = cur;
            z.xseq = p.st->xseq;
            *p.st = z;
        }
        if (blockIdx.x == 0 && grouped) {
            if (lane == 0) {
                Mailbox *mb = p.comm.box[p.comm.rank];
                mb->ll_seq = (unsigned long long)(ll_base + epoch);
                if (epoch >= 1u) mb->fused_hw[(ll_base + 1u) & 1u] = gridDim.x;     // what this solve left in each buffer
                if (epoch >= 2u) mb->fused_hw[(ll_base + 2u) & 1u] = gridDim.x;
            }
        }
        return;
    }

    if (warp == pcw + 1) {
        // ================================ comm warp (shared-step groups only) ===========================
        // mirrors the sequence of exchanges: per exchange, gather every peer's partials, then wait for the decision
        unsigned epoch = 0;
        double t_cur = p.t_start, dt;
        if (p.have_first_step) {
            dt = p.first_step;
        } else {
            remote_gather<1>(p, sh, ll_base + (++epoch));
            named_sync(kBarDecision, nthreads);
            Partial tot;
            tot.v[0] = sh.tot.a;
            tot.v[1] = __longlong_as_double((long long)sh.tot.b);
            tot.v[2] = tot.v[3] = 0.0;
            T d1max;
            const T h0 = init_h0<T>(p.c, &tot, 1, &d1max);
            remote_gather<1>(p, sh, ll_base + (++epoch));
            named_sync(kBarDecision, nthreads);
            tot.v[0] = sh.tot.a;
            dt = (double)init_dt<T>(p.c, &tot, 1, h0, d1max);
        }
        int done = (n_out <= 1) ? 1 : 0;
        if (!done && step_underflows(t_cur, dt)) done = 1;
        while (!done) {
            remote_gather<0>(p, sh, ll_base + (++epoch));
            named_sync(kBarDecision, nthreads);
            done = sh.ctl.done;
        }
        return;
    }

    // ================================ compute warps ====================================================
    long long i[TPT];                 // this thread's trajectories: lane `lane` of trajectory warps vw[u] = warp + u * pcw
    int vw[TPT];
    bool live[TPT];
#pragma unroll
    for (int u = 0; u < TPT; ++u) {
        vw[u] = warp + u * pcw;
        i[u] = (long long)blockIdx.x * (ncw * 32) + vw[u] * 32 + lane;
        live[u] = vw[u] < ncw && i[u] < p.n_traj;
    }
    const long long N = p.n_traj * D;
    const T *y0g = (const T *)p.y0;
    T *out = (T *)p.out;
    const bool rev = (T)p.time_sign < T(0);
    T y[TPT][D], f0[TPT][D];
#pragma unroll
    for (int u = 0; u < TPT; ++u) {
#pragma unroll
        for (int d = 0; d < D; ++d) y[u][d] = live[u] ? y0g[i[u] * D + d] : T(0);
        if (live[u]) {
#pragma unroll
            for (int d = 0; d < D; ++d) out[i[u] * D + d] = y[u][d];        // solution[0] = y0 (solvers.py:29)
        }
    }
    // The reverse-time wrapper of misc.py:318-321 is f'(t, y) = -f(-t, y).  The k's, f0 and f1 below hold f(-t, y) WITHOUT the
    // minus sign: every use multiplies a k by a value that is the same in every thread (the stage constants, the dense-output
    // constants, dtk, hk), and that value carries the sign instead.  Round-to-nearest is symmetric, so (-c)·k == c·(-k) bit for
    // bit, zeros and infinities included; the initial-step heuristic only squares f0 / scale and (f1 - f0) / scale.
    auto rhs = [&](T t, const T(&yy)[D], T(&dy)[D]) { RHS::eval(p.rhs, sw, rev ? -t : t, yy, dy); };
    // the barrier counts nthreads and nloc, re-derived at every barrier (see ntid_fresh).  Not for the 14-k tableaus: they do not
    // spill, and the registers it frees would change the co-resident capacity of fp64 Lorenz (170 -> 168 registers crosses an
    // allocation step), hence which batches take this kernel.
    auto bar_all = [&]() { return S <= 7 ? ntid_fresh() : nthreads; };
    auto bar_loc = [&]() { return S <= 7 ? ntid_fresh() - (p.comm.nranks > 1 ? 32 : 0) : nloc; };
    // hand each trajectory warp's share to the control warp; do not wait
    auto contribute = [&](const auto &mine, auto mode) {
        constexpr int MODE = decltype(mode)::value;
        Pay w[TPT];
#pragma unroll
        for (int u = 0; u < TPT; ++u) w[u] = pay_warp_reduce<MODE>(mine[u]);
        if (lane == 0) {
            // (vw recomputed from the block shape, like the barrier counts: kept in registers it is spilled)
            const int pcw_f = TPT > 1 ? (ntid_fresh() >> 5) - (p.comm.nranks > 1 ? 2 : 1) : pcw;
#pragma unroll
            for (int u = 0; u < TPT; ++u) {
                const int v = warp + u * pcw_f;
                if (v < ncw) sh.part[v] = w[u];
            }
        }
        named_arrive(kBarPartials, bar_loc());
    };
    double t_cur = p.t_start;
#pragma unroll
    for (int u = 0; u < TPT; ++u) rhs((T)t_cur, y[u], f0[u]);                 // dopri5.py:71

    // ---- first step: given (dopri5.py:76) or _select_initial_step (misc.py:183-247) ----------------------
    double dt;
    if (p.have_first_step) {
        dt = p.first_step;
    } else {
        const T rtol = (T)p.tab.rtol0, atol = (T)p.tab.atol0;
        T scale[TPT][D];
        Pay mine[TPT];
#pragma unroll
        for (int u = 0; u < TPT; ++u) {
            mine[u] = pay_identity<1>();
            double s0, s1;
            init_sums<T, D>(y[u], f0[u], rtol, atol, scale[u], s0, s1, live[u]);
            mine[u].a = s0;
            mine[u].b = (unsigned long long)__double_as_longlong(s1);
        }
        contribute(mine, IC<1>{});
        named_sync(kBarDecision, nthreads);
        Partial tot;
        tot.v[0] = sh.tot.a;
        tot.v[1] = __longlong_as_double((long long)sh.tot.b);
        tot.v[2] = tot.v[3] = 0.0;
        T d1max;
        const T h0 = init_h0<T>(p.c, &tot, 1, &d1max), hk = negate_if(h0, rev);
#pragma unroll
        for (int u = 0; u < TPT; ++u) {
            T y1[D], f1[D];
#pragma unroll
            for (int d = 0; d < D; ++d) y1[d] = A::add(y[u][d], A::mul(hk, f0[u][d]));
            rhs(A::add((T)t_cur, h0), y1, f1);
            double s2 = 0.0;
            if (live[u]) s2 = init_s2<T, D>(f1, f0[u], scale[u]);
            mine[u].a = s2;
            mine[u].b = 0ull;
        }
        contribute(mine, IC<1>{});
        named_sync(kBarDecision, nthreads);
        tot.v[0] = sh.tot.a;
        dt = (double)init_dt<T>(p.c, &tot, 1, h0, d1max);
    }
    int cur = 1;
    int done = (n_out <= 1) ? 1 : 0;
    if (!done && step_underflows(t_cur, dt)) done = 1;
    named_sync(kBarFirstStep, nloc);                                       // the first attempt's stage constants are in ssc

    // ---- attempts -------------------------------------------------------------------------------------
    using SC = StageConst<T, S>;
    int att = 0;
    while (!done) {
        const T t0c = (T)t_cur, dtc = (T)dt;                               // rk_common.py:45-46
        const T dtk = negate_if(dtc, rev);                                 // dt with the sign of the k's (see `rhs`)
        T k[S][TPT][D];
#pragma unroll
        for (int u = 0; u < TPT; ++u)
#pragma unroll
            for (int d = 0; d < D; ++d) k[0][u][d] = f0[u][d];
        auto kj = [&](int j, int u, int d) { return k[j][u][d]; };
        T yi[TPT][D];
#pragma unroll
        for (int s = 0; s < S - 1; ++s) {
            const T ti = A::add(t0c, A::mul((T)p.c.alpha[s], dtc));
            T acc[TPT][D];
            tableau_combine<T>(acc, s + 1, [&](int j) { return ssc.c[SC::beta(s, j)]; }, kj);   // dt·beta (scale * x)
#pragma unroll
            for (int u = 0; u < TPT; ++u) {
#pragma unroll
                for (int d = 0; d < D; ++d) yi[u][d] = A::add(y[u][d], acc[u][d]);
                rhs(ti, yi[u], k[s + 1][u]);
            }
        }
        if (!p.tab.fsal) {                                                 // rk_common.py:54-56
            T acc[TPT][D];
            tableau_combine<T>(acc, S, [&](int j) { return ssc.c[SC::sol(j)]; }, kj);
#pragma unroll
            for (int u = 0; u < TPT; ++u)
#pragma unroll
                for (int d = 0; d < D; ++d) yi[u][d] = A::add(y[u][d], acc[u][d]);
        }
        // error estimate + this thread's share of the reduction (rk_common.py:60, misc.py:256-263)
        {
            Pay mine[TPT];
            T err[TPT][D];
            tableau_combine<T>(err, S, [&](int j) { return ssc.c[SC::err(j)]; }, kj);
#pragma unroll
            for (int u = 0; u < TPT; ++u) {
                mine[u] = pay_identity<0>();
                if (live[u]) {
                    const NormTerms nt = norm_terms<T, D>(err[u], y[u], yi[u]);
                    mine[u].a = nt.ssq;
                    mine[u].b = nt.amax;
                    mine[u].flag = nt.bad0 ? 1u : 0u;
                }
            }
            contribute(mine, IC<0>{});
        }
        FTRACE(att, 8);
        // ---- dense output (dopri5.py:39-45, interp.py:22-67): the VALUES of the first kDenseRows output rows of the step are
        // computed now, while the control warp runs the reduction (the arithmetic overlaps the exchange latency); they are
        // STORED only once the step is known to be accepted -- the stores then drain under the next attempt's stages instead
        // of queueing in front of the control warp's loads (measured: speculative stores tripled the exchange time)
        const double t1_acc = t_cur + dt;
        const int c2 = next_cursor(t_out, cur, n_out, t1_acc);
        const T t0s = t0c, t1s = (T)t1_acc;
        auto fit = [&](int u, const DenseConst<T, S> &dc, T(&ca)[D], T(&cb)[D], T(&cc)[D], T(&cd)[D]) {
            T ymid[D];
            {
                T acc[1][D];
                tableau_combine<T>(acc, S, [&](int j) { return dc.cmid[j]; }, [&](int j, int, int d) { return k[j][u][d]; });
#pragma unroll
                for (int d = 0; d < D; ++d) ymid[d] = A::add(y[u][d], acc[0][d]);
            }
#pragma unroll
            for (int d = 0; d < D; ++d)
                quartic_fit<T, S>(dc, dtk, k[0][u][d], k[S - 1][u][d], y[u][d], yi[u][d], ymid[d], ca[d], cb[d], cc[d], cd[d]);
        };
        auto eval_x = [&](int u, T x, T x2, T x3, T x4, const T(&ca)[D], const T(&cb)[D], const T(&cc)[D], const T(&cd)[D],
                          T(&r)[D]) {
#pragma unroll
            for (int d = 0; d < D; ++d) r[d] = quartic_eval<T>(ca[d], cb[d], cc[d], cd[d], y[u][d], x, x2, x3, x4);
        };
        // the rows wait in shared memory, laid out exactly like the block's contiguous chunk of an output row
        const bool blk_out = c2 > cur;                                        // uniform over the grid
        if (blk_out) {
            named_sync(kBarRows, bar_loc());                              // the control warp has copied the previous step's rows out
#pragma unroll
            for (int u = 0; u < TPT; ++u) {                               // (one trajectory after the other: fewer live registers)
                if (live[u]) {
                    T ca[D], cb[D], cc[D], cd[D];
                    fit(u, sdc.k, ca, cb, cc, cd);
#pragma unroll
                    for (int q = 0; q < kDenseRows; ++q) {
                        if (cur + q < c2) {
                            T r[D];
                            eval_x(u, sdc.x[q][0], sdc.x[q][1], sdc.x[q][2], sdc.x[q][3], ca, cb, cc, cd, r);
#pragma unroll
                            for (int d = 0; d < D; ++d) s_rows[q][(vw[u] * 32 + lane) * D + d] = r[d];
                        }
                    }
                }
            }
        }
        if (blk_out) named_arrive(kBarRowsReady, bar_loc());              // rows handed to the control warp
        FTRACE(att, 9);
        named_sync(kBarDecision, bar_all());                                // the control warp's decision
        const bool accept = sh.ctl.accept != 0;
        FTRACE_DEP(att, 10, sh.ctl.accept);
        // state update (dopri5.py:113-120)
        if (accept) {
            if (blk_out && cur + kDenseRows < c2) {
                // long steps: the remaining rows, after the fact, with constants of their own (the control warp is already
                // overwriting sdc for the next attempt)
                const DenseConst<T, S> dc = dense_const<T, S>(p.tab, dtk);
                const T den = A::sub(t1s, t0s);
#pragma unroll
                for (int u = 0; u < TPT; ++u) {
                    if (!live[u]) continue;
                    T ca[D], cb[D], cc[D], cd[D];
                    fit(u, dc, ca, cb, cc, cd);                              // (recomputed: not kept live over the barrier)
                    for (int j = cur + kDenseRows; j < c2; ++j) {
                        const T x = A::div(A::sub((T)__ldg(t_out + j), t0s), den);
                        const T x2 = A::mul(x, x), x3 = A::mul(x2, x), x4 = A::mul(x3, x);
                        T r[D];
                        eval_x(u, x, x2, x3, x4, ca, cb, cc, cd, r);
                        T *row = out + (long long)j * N + i[u] * D;
#pragma unroll
                        for (int d = 0; d < D; ++d) row[d] = r[d];
                    }
                }
            }
            t_cur = t1_acc;
            cur = c2;                     // (a non-finite y0 also sets `done`, so the cursor is moot in that case)
#pragma unroll
            for (int u = 0; u < TPT; ++u)
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    y[u][d] = yi[u][d];
                    f0[u][d] = k[S - 1][u][d];
                }
        }
        dt = sh.ctl.dt_next;
        done = sh.ctl.done;
        ++att;
    }
}

// ================================================================================================
// host side
// ================================================================================================
// What fused_launch needs to know of the device for one instantiation, queried once per process and device: cooperative
// launch support, the SM count, and how many blocks of w warps the occupancy calculator puts on an SM.  (Every solve asks
// for the capacity and the geometry; the occupancy queries behind them would otherwise cost more than the launch.)
struct FusedDevInfo {
    bool ready;
    int coop, nsm;
    int per_sm[33];       // [warps per block]
};
constexpr int kFusedMaxDevices = 64;

template <typename T, typename RHS, int S, int MAXT>
static int fused_dev_info(const FusedDevInfo **out) {
    static std::mutex mu;
    static FusedDevInfo info[kFusedMaxDevices];
    int dev = 0;
    B2_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= kFusedMaxDevices) return b2_fail(B2ODE_EINVAL, "device ordinal %d out of range", dev);
    std::lock_guard<std::mutex> lock(mu);
    FusedDevInfo &d = info[dev];
    if (!d.ready) {
        B2_CUDA(cudaDeviceGetAttribute(&d.coop, cudaDevAttrCooperativeLaunch, dev));
        B2_CUDA(cudaDeviceGetAttribute(&d.nsm, cudaDevAttrMultiProcessorCount, dev));
        for (int w = 2; w <= FusedShape<T, RHS, S, MAXT>::threads / 32; ++w)
            B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d.per_sm[w], k_fused_adaptive<T, RHS, S, MAXT>, 32 * w, 0));
        d.ready = true;
    }
    *out = &d;
    return 0;
}

// Block geometry in trajectory warps (NCW, 32 trajectories each; ceil(NCW / TPT) compute warps) + the service warps.  One
// block per SM when the batch allows it (fewest partials to gather, every SM busy): NCW = ceil(ceil(n / SMs) / 32),
// capped by the register budget of the instantiation; if that does not keep the batch co-resident, the largest block that
// does (smaller blocks can pack more warps per SM when the register file, not the block size, is the limit).  A pure
// function of (n, device, instantiation): every rank of a shared-step group computes the same geometry for every other
// rank's shard.
template <int MAXT, int TPT>
static int fused_geometry(const FusedDevInfo &di, long long n_traj, int nsvc, int *ncw_out, int *grid_out) {
    const int nsm = di.nsm;
    const int kMaxNcw = MAXT / 32 - nsvc;
    long long per_block = (n_traj + nsm - 1) / nsm;
    int ncw = (int)((per_block + 31) / 32);
    if (ncw < 1) ncw = 1;
    if (ncw > kMaxNcw) ncw = kMaxNcw;
    for (; ncw >= 1; --ncw) {
        const int grid = (int)((n_traj + (long long)ncw * 32 - 1) / ((long long)ncw * 32));
        if (grid <= di.per_sm[fused_warps(ncw, TPT, nsvc)] * nsm) {
            *ncw_out = ncw;
            *grid_out = grid;
            return 0;
        }
    }
    return b2_fail(B2ODE_ENOMEM, "batch of %lld trajectories cannot stay co-resident on %d SMs", n_traj, nsm);
}

// `capacity` != null: only report how many trajectories this instantiation can keep co-resident on the current device.
// n_traj_rank: trajectories of every rank of the group (null / ignored without a group).
template <typename T, typename RHS, int S, int MAXT>
static int fused_launch(const FusedParams &p_in, long long n_traj, cudaStream_t st, long long *capacity, const int64_t *n_traj_rank) {
    constexpr int TPT = FusedShape<T, RHS, S, MAXT>::tpt;
    const FusedDevInfo *di = nullptr;
    {
        const int rc = fused_dev_info<T, RHS, S, MAXT>(&di);
        if (rc) return rc;
    }
    if (capacity) {
        // (reported for the geometry with both service warps, so that a batch that fits alone also fits in a group)
        long long best = 0;
        for (int ncw = MAXT / 32 - 2; ncw >= 1 && di->coop; --ncw) {
            const long long cap = (long long)di->per_sm[fused_warps(ncw, TPT, 2)] * di->nsm * ncw * 32;
            if (cap > best) best = cap;
        }
        *capacity = best;
        return 0;
    }
    if (!di->coop) return b2_fail(B2ODE_ESTATE, "device does not support cooperative launch");
    FusedParams p = p_in;
    const int nsvc = p.comm.nranks > 1 ? 2 : 1;        // control warp (+ comm warp with a shared-step group)
    int ncw = 0, grid = 0;
    {
        const int rc = fused_geometry<MAXT, TPT>(*di, n_traj, nsvc, &ncw, &grid);
        if (rc) return rc;
    }
    if (p.comm.nranks > 1) {
        for (int r = 0; r < p.comm.nranks; ++r) {
            int ncw_r = 0, grid_r = 0;
            const int rc = fused_geometry<MAXT, TPT>(*di, n_traj_rank[r], nsvc, &ncw_r, &grid_r);
            if (rc) return rc;
            if (grid_r > kMaxFusedBlocks)
                return b2_fail(B2ODE_ENOMEM, "rank %d needs %d blocks, the group mailbox holds %d", r, grid_r, kMaxFusedBlocks);
            p.comm.grid_of[r] = grid_r;
        }
        if (p.comm.grid_of[p.comm.rank] != grid) return b2_fail(B2ODE_ESTATE, "inconsistent shard size for this rank");
    }
    p.ncw = ncw;
    void *args[] = {(void *)&p};
    const int slot = b2_timing_begin(6 /* B2_FAM_FUSED */, st);
    B2_CUDA(cudaLaunchCooperativeKernel((const void *)k_fused_adaptive<T, RHS, S, MAXT>, dim3(grid),
                                        dim3(32 * fused_warps(ncw, TPT, nsvc)), args, 0, st));
    b2_timing_end(6, slot, st);
    b2_count_launch();
    return 0;
}

// f(std::integral_constant<int, S>{}) for the stage counts every kernel family here is instantiated for; `what` names the
// entry point in the refusal of any other count
template <typename F>
static int dispatch_nk(const char *what, int n_k, F &&f) {
    return dispatch_count(std::integer_sequence<int, 2, 4, 7, 14>{}, n_k, f, "%s supports tableaus with 2, 4, 7 or 14 k's (got %d)",
                          what, n_k);
}

// dispatch_nk's refusal, for entry points that check the tableau before any CUDA call
static int check_nk(const char *what, int n_k) {
    return dispatch_nk(what, n_k, [](auto) { return 0; });
}

template <typename T>
static int fused_dispatch_rhs(const FusedParams &p, int rhs_kind, int n_k, long long n_traj, cudaStream_t st,
                              long long *capacity = nullptr, const int64_t *ntr = nullptr) {
    // trajectory budget per block: 512 threads' worth (<= 128 registers per thread at one trajectory per thread) for the
    // 2- and 4-k tableaus, 256 for 14 k's.  The 7-k tableaus (dopri5) take 576 threads' worth: 17 trajectory warps alone, 16
    // in a group, so one block per SM holds 132 x 512 = 67 584 trajectories on an H100, config 2's 65 536 included.  At two
    // trajectories per thread (FusedShape) that is 8 or 9 compute warps + the service warps (<= 320 threads, <= 168
    // registers).  The fp64 latent MLP takes 256 threads' worth everywhere: its 10.8 KB of weights next to 3 dense-output
    // rows of 17 trajectory warps overflow the 48 KB of static shared memory, and at 576 (512) threads' worth its stage
    // phase spills under the 96- (128-) register cap.
    return dispatch_rhs<T>(rhs_kind, [&](auto rhs) {
        using RHS = decltype(rhs);
        return dispatch_nk("fused solve", n_k, [&](auto s) {
            constexpr int S = decltype(s)::value;
            constexpr bool narrow = std::is_same<RHS, RhsLatentMLP<double>>::value;
            constexpr int MAXT = (S == 14 || narrow) ? 256 : S == 7 ? 576 : 512;
            return fused_launch<T, RHS, S, MAXT>(p, n_traj, st, capacity, ntr);
        });
    });
}

// Largest batch (trajectories on this device) b2ode_fused_solve can keep co-resident for this tableau / dtype / right-hand
// side: the host asks BEFORE launching, so that the shards of a shared-step group can agree on one path.  < 0: error.
extern "C" int64_t b2ode_fused_capacity(const b2ode_adaptive_desc *desc, int rhs_kind) {
    if (!desc) return b2_fail(B2ODE_EINVAL, "null argument");
    FusedParams p;
    memset(&p, 0, sizeof(p));
    long long cap = 0;
    int rc;
    if (desc->dtype == B2ODE_F64) rc = fused_dispatch_rhs<double>(p, rhs_kind, desc->n_k, 0, nullptr, &cap);
    else if (desc->dtype == B2ODE_F32) rc = fused_dispatch_rhs<float>(p, rhs_kind, desc->n_k, 0, nullptr, &cap);
    else return b2_fail(B2ODE_EINVAL, "dtype must be 0 or 1");
    if (rc) return rc < 0 ? rc : -rc;
    return (int64_t)cap;
}

extern "C" size_t b2ode_fused_workspace_bytes(int64_t n_traj) {
    const long long grid_max = (n_traj + 31) / 32;       // the smallest block has one compute warp
    // [arrival counter, 128 B][row progress counter, 128 B][partials 2 x grid x 16 B (no shared-step group)]
    return (size_t)256 + (size_t)grid_max * 32;
}

extern "C" int b2ode_fused_solve(const b2ode_adaptive_desc *desc, const b2ode_fused_desc *f) {
    if (!desc || !f) return b2_fail(B2ODE_EINVAL, "null argument");
    if (!f->y0 || !f->out || !f->t_out || !f->state || !f->workspace) return b2_fail(B2ODE_EINVAL, "null buffer");
    if (desc->nseg != 1) return b2_fail(B2ODE_EINVAL, "fused solve takes a single-tensor state");
    long long n_traj = 0;
    {
        const int rc = check_rhs(&f->rhs, desc->seg_len[0], &n_traj);
        if (rc) return rc;
    }
    const int D = rhs_row_dim(f->rhs.kind);
    if (desc->dense_kind != 0) return b2_fail(B2ODE_EINVAL, "fused solve supports the quartic dense output only");
    if (n_traj < 1) return b2_fail(B2ODE_EINVAL, "empty batch");
    if (f->workspace_bytes < b2ode_fused_workspace_bytes(n_traj)) return b2_fail(B2ODE_ENOMEM, "workspace too small");
    cudaStream_t st = (cudaStream_t)f->cuda_stream;
    unsigned char *w = (unsigned char *)f->workspace;
    if ((uintptr_t)w & 15u) return b2_fail(B2ODE_EINVAL, "workspace must be 16-byte aligned");
    const int nranks = f->nranks > 1 ? f->nranks : 1;
    FusedParams p;
    memset(&p, 0, sizeof(p));
    B2_CUDA(cudaMemsetAsync(w, 0, 256, st));
    p.progress = (unsigned *)(w + 128);
    p.host_mark = (int *)f->host_mark;
    p.st = (b2ode_state *)f->state;
    p.y0 = f->y0;
    p.out = f->out;
    p.n_traj = n_traj;
    p.have_first_step = (f->first_step == f->first_step) ? 1 : 0;
    p.t_start = f->t_start;
    p.first_step = f->first_step;
    fill_rhs(p, f->rhs);
    fill_tableau(p.tab, *desc);
    fill_ctrl(p.c, *desc);
    p.c.n_out = f->n_out;
    p.c.t_out = f->t_out;
    long long n_glob = n_traj;
    p.comm.rank = 0;
    p.comm.nranks = 0;
    if (nranks > 1) {
        if (!f->mailboxes || nranks > B2ODE_MAXPEERS || f->rank < 0 || f->rank >= nranks) return b2_fail(B2ODE_EINVAL, "bad group arguments");
        n_glob = 0;
        for (int r = 0; r < nranks; ++r) {
            if (!f->mailboxes[r] || f->n_traj_rank[r] < 1) return b2_fail(B2ODE_EINVAL, "bad mailbox / shard size of rank %d", r);
            n_glob += f->n_traj_rank[r];
            p.comm.box[r] = (Mailbox *)f->mailboxes[r];
        }
        if (f->n_traj_rank[f->rank] != n_traj) return b2_fail(B2ODE_EINVAL, "n_traj_rank[rank] does not match the state");
        p.comm.rank = f->rank;
        p.comm.nranks = nranks;
    }
    // intra-GPU receive area = the caller's workspace: [arrival counter][row progress][partials 2 x grid x 16 B], zeroed per launch
    B2_CUDA(cudaMemsetAsync(w + 256, 0, b2ode_fused_workspace_bytes(n_traj) - 256, st));
    p.ctr = (unsigned *)w;
    p.part2 = (unsigned long long *)(w + 256);
    p.c.n_global[0] = n_glob * D;
    if (desc->dtype == B2ODE_F64) return fused_dispatch_rhs<double>(p, f->rhs.kind, desc->n_k, n_traj, st, nullptr, f->n_traj_rank);
    if (desc->dtype == B2ODE_F32) return fused_dispatch_rhs<float>(p, f->rhs.kind, desc->n_k, n_traj, st, nullptr, f->n_traj_rank);
    return b2_fail(B2ODE_EINVAL, "dtype must be 0 or 1");
}

// ================================================================================================
// fixed-grid methods with a built-in right-hand side: no step-size control, hence no reductions at all --
// every thread integrates its trajectory through the whole grid and writes its outputs
// (tfdiffeq/solvers.py:82-115, fixed_grid.py, rk_common.py:73-81; same operation order as k_fixed<T, OP>)
// ================================================================================================
struct FusedFixedParams {
    const void *y0;
    void *out;
    long long n_traj;
    int n_steps, n_out, method;     // method: 0 euler, 1 midpoint, 2 heun, 3 rk4 (3/8 rule)
    const void *times;              // [n_steps][4] stage times, state dtype
    const void *dts;                // [n_steps]
    const int *j0;                  // [n_steps + 1]: outputs inside cell i are [j0[i], j0[i+1])
    const unsigned char *ends;      // [n_steps]: the cell ends exactly on its last output
    const void *s1;                 // [n_steps]  t1 - t0
    const void *s2;                 // [n_out]    t_out[j] - t0 of its cell
    double time_sign;
    double rhs[8];
    const void *rhs_data;
};

template <typename T, typename RHS>
__global__ void __launch_bounds__(256) k_fused_fixed(const __grid_constant__ FusedFixedParams p) {
    using A = Ar<T>;
    constexpr int D = RHS::D;
    __shared__ T sw[RHS::kSmem];
    stage_weights<T, RHS>(p.rhs, p.rhs_data, sw, 256);
    const T tsign = (T)p.time_sign;
    auto rhs = [&](T t, const T(&yy)[D], T(&dy)[D]) {
        if (tsign < T(0)) {
            RHS::eval(p.rhs, sw, -t, yy, dy);
#pragma unroll
            for (int d = 0; d < D; ++d) dy[d] = -dy[d];
        } else {
            RHS::eval(p.rhs, sw, t, yy, dy);
        }
    };
    const long long N = p.n_traj * D;
    const T *times = (const T *)p.times, *dts = (const T *)p.dts, *s1 = (const T *)p.s1, *s2 = (const T *)p.s2;
    T *out = (T *)p.out;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < p.n_traj; i += (long long)gridDim.x * 256) {
        T y[D];
#pragma unroll
        for (int d = 0; d < D; ++d) {
            y[d] = ((const T *)p.y0)[i * D + d];
            out[i * D + d] = y[d];
        }
        for (int s = 0; s < p.n_steps; ++s) {
            const T dt = dts[s];
            const T *tm = times + 4 * s;
            T y1[D], k1[D], k2[D], k3[D], k4[D], ys[D];
            rhs(tm[0], y, k1);
            if (p.method == 0) {
#pragma unroll
                for (int d = 0; d < D; ++d) y1[d] = A::add(y[d], A::mul(dt, k1[d]));                       // B2ODE_OP_EULER
            } else if (p.method == 1) {
#pragma unroll
                for (int d = 0; d < D; ++d) ys[d] = A::add(y[d], A::div(A::mul(k1[d], dt), T(2)));         // HALF_STEP
                rhs(tm[1], ys, k2);
#pragma unroll
                for (int d = 0; d < D; ++d) y1[d] = A::add(y[d], A::mul(dt, k2[d]));
            } else if (p.method == 2) {
#pragma unroll
                for (int d = 0; d < D; ++d) ys[d] = A::add(y[d], A::mul(dt, k1[d]));
                rhs(tm[1], ys, k2);
#pragma unroll
                for (int d = 0; d < D; ++d) y1[d] = A::add(y[d], A::mul(A::div(dt, T(2)), A::add(k1[d], k2[d])));   // HEUN_FINAL
            } else {
#pragma unroll
                for (int d = 0; d < D; ++d) ys[d] = A::add(y[d], A::div(A::mul(dt, k1[d]), T(3)));         // RK4_S2
                rhs(tm[1], ys, k2);
#pragma unroll
                for (int d = 0; d < D; ++d) ys[d] = A::add(y[d], A::mul(dt, A::add(A::div(k1[d], T(-3)), k2[d])));   // RK4_S3
                rhs(tm[2], ys, k3);
#pragma unroll
                for (int d = 0; d < D; ++d) ys[d] = A::add(y[d], A::mul(dt, A::add(A::sub(k1[d], k2[d]), k3[d])));   // RK4_S4
                rhs(tm[3], ys, k4);
#pragma unroll
                for (int d = 0; d < D; ++d)
                    y1[d] = A::add(y[d], A::mul(A::add(A::add(A::add(k1[d], A::mul(T(3), k2[d])), A::mul(T(3), k3[d])), k4[d]),
                                                A::div(dt, T(8))));                                          // RK4_FINAL
            }
            const int ja = p.j0[s], jb = p.j0[s + 1];
            for (int j = ja; j < jb; ++j) {
                T *row = out + (long long)j * N + i * D;
                if (j == jb - 1 && p.ends[s]) {
#pragma unroll
                    for (int d = 0; d < D; ++d) row[d] = y1[d];
                } else {
#pragma unroll
                    for (int d = 0; d < D; ++d) row[d] = A::add(y[d], A::mul(A::div(A::sub(y1[d], y[d]), s1[s]), s2[j]));   // LERP
                }
            }
#pragma unroll
            for (int d = 0; d < D; ++d) y[d] = y1[d];
        }
    }
}

template <typename T>
static int fused_fixed_dispatch(const FusedFixedParams &p, int rhs_kind, int sm_count, cudaStream_t st) {
    const int grid = (int)capped_grid(p.n_traj, 256, 8, sm_count);
    return dispatch_rhs<T>(rhs_kind, [&](auto rhs) {
        k_fused_fixed<T, decltype(rhs)><<<grid, 256, 0, st>>>(p);
        B2_CUDA(cudaGetLastError());
        b2_count_launch();
        return 0;
    });
}

extern "C" int b2ode_fused_fixed_solve(int dtype, int method, const b2ode_rhs_desc *rhs, const void *y0, void *out,
                                       int64_t n_traj, int n_steps, int n_out, const void *times, const void *dts,
                                       const int32_t *j0, const unsigned char *ends, const void *s1, const void *s2,
                                       int sm_count, void *cuda_stream) {
    if (!y0 || !out || n_traj < 1 || n_out < 1 || n_steps < 0) return b2_fail(B2ODE_EINVAL, "bad arguments");
    if (n_steps > 0 && (!times || !dts || !j0 || !ends || !s1 || !s2)) return b2_fail(B2ODE_EINVAL, "null grid array");
    if (method < 0 || method > 3) return b2_fail(B2ODE_EINVAL, "method must be 0..3");
    long long rows = 0;   // == n_traj: the state is whole rows by construction
    const int rc = check_rhs(rhs, rhs ? n_traj * rhs_row_dim(rhs->kind) : 0, &rows);
    if (rc) return rc;
    FusedFixedParams p;
    memset(&p, 0, sizeof(p));
    p.y0 = y0;
    p.out = out;
    p.n_traj = n_traj;
    p.n_steps = n_steps;
    p.n_out = n_out;
    p.method = method;
    p.times = times;
    p.dts = dts;
    p.j0 = j0;
    p.ends = ends;
    p.s1 = s1;
    p.s2 = s2;
    fill_rhs(p, *rhs);
    if (dtype == B2ODE_F64) return fused_fixed_dispatch<double>(p, rhs->kind, sm_count, (cudaStream_t)cuda_stream);
    if (dtype == B2ODE_F32) return fused_fixed_dispatch<float>(p, rhs->kind, sm_count, (cudaStream_t)cuda_stream);
    return b2_fail(B2ODE_EINVAL, "dtype must be 0 or 1");
}

// ================================================================================================
// independent rows (DESIGN.md §4.2(c)): every row of the state -- RHS::D consecutive elements -- is its own ODE system with
// its own step size, error norm and output cursor, solved as if it had been passed to the persistent kernel alone.  One row
// per thread, state, f0 and all s k's in registers; no reduction, no barrier inside the solve, no co-residency requirement.
// The arithmetic is the persistent kernel's (tableau_combine with dt·beta carrying the sign of the time direction, the norm
// terms, the initial-step sums, quartic_fit / quartic_eval) with the controller of the stage kernels (ctrl_decide, one
// segment of D elements).  The norm terms, each initial-step sum and the bookkeeping are written out here, in the operations
// and order of norm_terms, init_sums, init_s2 and advance_step: called through its helper, each one alone moves this
// kernel's machine code.
// ================================================================================================
struct RowsParams {
    const void *y0;
    void *out;
    long long n_rows;
    unsigned long long *next;          // row hand-out counter, zeroed before the launch
    long long *n_acc, *n_rej;          // per row
    double *dt_next, *error_ratio;
    int *status;
    int have_first_step;
    double t_start, first_step;
    double time_sign;                  // -1 when integrating the reversed system (misc.py:318-321)
    double rhs[8];
    const void *rhs_data;
    Tableau tab;
    CtrlParams c;                      // n_global[0] = D: the mean of the error norm is over one row
    // recording variant only (b2ode_rows_solve_record): every accepted step n < rec_cap of row r writes y_n, (t_n, dt_n)
    // and, without FSAL, f0 into slot n, slot-major ([slot][row][D]; see b2ode_rows_record_desc)
    void *rec_y, *rec_f0;
    double *rec_t;
    long long rec_cap;
};

// Threads per block (ptxas -v, DESIGN.md §4.2(c)): 128 everywhere; the bound leaves each instantiation the registers it asks
// for (dopri8 fp64 Kepler: 14 k's x 4 doubles) and the occupancy calculator then sizes the grid.
template <typename T, typename RHS, int S>
struct RowsShape {
    static constexpr int threads = 128;
};

// REC: the recording variant for the backward pass (b2ode_rows_solve_record): the same arithmetic plus the stores of an
// accepted step's start; REC = false compiles to the plain solve.
template <typename T, typename RHS, int S, bool REC>
__global__ void __launch_bounds__(RowsShape<T, RHS, S>::threads) k_rows_adaptive(const __grid_constant__ RowsParams p) {
    using A = Ar<T>;
    constexpr int D = RHS::D;
    __shared__ T sw[RHS::kSmem];
    stage_weights<T, RHS>(p.rhs, p.rhs_data, sw, blockDim.x);
    // the k's hold f(-t, y) without the minus sign in reverse time; the dt factors that multiply them carry it (see `rhs` in
    // k_fused_adaptive)
    const bool rev = (T)p.time_sign < T(0);
    auto rhs = [&](T t, const T(&yy)[D], T(&dy)[D]) { RHS::eval(p.rhs, sw, rev ? -t : t, yy, dy); };
    const int n_out = p.c.n_out;
    const double *__restrict__ t_out = p.c.t_out;
    const long long N = p.n_rows * D;
    const T *y0g = (const T *)p.y0;
    T *out = (T *)p.out;
    // rows are handed out dynamically: a thread that finishes its row takes the next one, so a warp does not wait for the
    // slowest of 32 fixed rows.  A row's result depends on that row alone, so the assignment changes no bit.
    const long long nthr = (long long)gridDim.x * blockDim.x;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < p.n_rows;
         r = nthr + (long long)atomicAdd(p.next, 1ull)) {
        T y[D], f0[D];
#pragma unroll
        for (int d = 0; d < D; ++d) {
            y[d] = y0g[r * D + d];
            out[r * D + d] = y[d];                                          // solution[0] = y0 (solvers.py:29)
        }
        double t_cur = p.t_start;
        rhs((T)t_cur, y, f0);                                               // dopri5.py:71
        double dt;
        if (p.have_first_step) {
            dt = p.first_step;                                              // dopri5.py:76
        } else {
            // _select_initial_step (misc.py:183-247) on this row's D elements
            const T rtol = (T)p.tab.rtol0, atol = (T)p.tab.atol0;
            T scale[D];
            double s0 = 0.0, s1 = 0.0;
#pragma unroll
            for (int d = 0; d < D; ++d) {
                scale[d] = A::add(atol, A::mul(A::abs(y[d]), rtol));
                const double q0 = (double)A::div(y[d], scale[d]), q1 = (double)A::div(f0[d], scale[d]);
                s0 += q0 * q0;
                s1 += q1 * q1;
            }
            Partial tot;
            tot.v[0] = s0;
            tot.v[1] = s1;
            tot.v[2] = tot.v[3] = 0.0;
            T d1max;
            const T h0 = init_h0<T>(p.c, &tot, 1, &d1max), hk = negate_if(h0, rev);
            T y1[D], f1[D];
#pragma unroll
            for (int d = 0; d < D; ++d) y1[d] = A::add(y[d], A::mul(hk, f0[d]));
            rhs(A::add((T)t_cur, h0), y1, f1);
            double s2 = 0.0;
#pragma unroll
            for (int d = 0; d < D; ++d) {
                const double q = (double)A::div(A::sub(f1[d], f0[d]), scale[d]);
                s2 += q * q;
            }
            tot.v[0] = s2;
            dt = (double)init_dt<T>(p.c, &tot, 1, h0, d1max);
        }
        unsigned status = 0u;
        int cur = 1;
        bool done = n_out <= 1;
        if (!done && step_underflows(t_cur, dt)) {
            status |= B2ODE_ST_UNDERFLOW;
            done = true;
        }
        double m_last = 0.0;
        long long n_acc = 0, n_rej = 0, nadv = 0;
        while (!done) {
            const T t0c = (T)t_cur, dtc = (T)dt;                           // rk_common.py:45-46
            const T dtk = negate_if(dtc, rev);                             // dt with the sign of the k's
            T k[S][D], yi[D];
#pragma unroll
            for (int d = 0; d < D; ++d) k[0][d] = f0[d];
            auto kj = [&](int j, int, int d) { return k[j][d]; };
#pragma unroll
            for (int s = 0; s < S - 1; ++s) {                              // rk_common.py:49-52
                const T ti = A::add(t0c, A::mul((T)p.c.alpha[s], dtc));
                T acc[1][D];
                tableau_combine<T>(acc, s + 1, [&](int j) { return A::mul(dtk, (T)p.tab.beta[s][j]); }, kj);   // dt·beta
#pragma unroll
                for (int d = 0; d < D; ++d) yi[d] = A::add(y[d], acc[0][d]);
                rhs(ti, yi, k[s + 1]);
            }
            if (!p.tab.fsal) {                                             // rk_common.py:54-56
                T acc[1][D];
                tableau_combine<T>(acc, S, [&](int j) { return A::mul(dtk, (T)p.tab.c_sol[j]); }, kj);
#pragma unroll
                for (int d = 0; d < D; ++d) yi[d] = A::add(y[d], acc[0][d]);
            }
            // error estimate (rk_common.py:60) and the row's norm terms in one pass, in element order (misc.py:256-263):
            // sum err^2 in fp64, max|y0| and max|y1| as bit patterns of non-negative doubles (NaN sorts above +inf)
            double sum = 0.0;
            unsigned long long m0 = 0ull, m1 = 0ull;
            {
                T err[1][D];
                tableau_combine<T>(err, S, [&](int j) { return A::mul(dtk, (T)p.tab.c_error[j]); }, kj);
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    const double ed = (double)err[0][d];
                    sum += ed * ed;
                    m0 = umax64(m0, (unsigned long long)__double_as_longlong(fabs((double)y[d])));
                    m1 = umax64(m1, (unsigned long long)__double_as_longlong(fabs((double)yi[d])));
                }
            }
            Partial tot;
            tot.v[0] = sum;
            tot.v[1] = tot.v[2] = __longlong_as_double((long long)umax64(m0, m1));
            tot.v[3] = (m0 >= 0x7ff0000000000000ull) ? 1.0 : 0.0;          // inf or NaN in y0 (dopri5.py:100)
            const CtrlDecision dec = ctrl_decide<T>(p.c, &tot, 1, dt);
            // advance() bookkeeping (dopri5.py:83-120): advance_step's rule, written out (see above)
            const double t1_acc = t_cur + dt;
            const int c2 = next_cursor(t_out, cur, n_out, t1_acc);
            unsigned st_bits = status | (dec.bad0 ? B2ODE_ST_NONFINITE : 0u);
            const bool adv = dec.accept && !dec.bad0;
            const double t1n = dec.accept ? t1_acc : t_cur;
            const int c_new = adv ? c2 : cur;
            const long long nadv2 = (c_new > cur) ? 0 : nadv + 1;
            bool dn = c_new >= n_out;
            if (!dn) {
                if (nadv2 >= p.c.max_num_steps) st_bits |= B2ODE_ST_MAXSTEPS;
                if (step_underflows(t1n, dec.dt_next)) st_bits |= B2ODE_ST_UNDERFLOW;
            }
            if (st_bits) dn = true;
            if (adv && c2 > cur) {
                // dense output of the accepted step (dopri5.py:39-45, interp.py:22-67), every output time in (t0, t1], in
                // the persistent kernel's operation order, stored straight to out[j, r, :]
                const DenseConst<T, S> dc = dense_const<T, S>(p.tab, dtk);
                const T t0s = t0c, den = A::sub((T)t1_acc, t0s);
                T ca[D], cb[D], cc[D], cd[D];
                {
                    T ymid[1][D];
                    tableau_combine<T>(ymid, S, [&](int j) { return dc.cmid[j]; }, kj);
#pragma unroll
                    for (int d = 0; d < D; ++d)
                        quartic_fit<T, S>(dc, dtk, k[0][d], k[S - 1][d], y[d], yi[d], A::add(y[d], ymid[0][d]), ca[d], cb[d], cc[d], cd[d]);
                }
                for (int j = cur; j < c2; ++j) {
                    const T x = A::div(A::sub((T)__ldg(t_out + j), t0s), den);
                    const T x2 = A::mul(x, x), x3 = A::mul(x2, x), x4 = A::mul(x3, x);
                    T *row = out + (long long)j * N + r * D;
#pragma unroll
                    for (int d = 0; d < D; ++d) row[d] = quartic_eval<T>(ca[d], cb[d], cc[d], cd[d], y[d], x, x2, x3, x4);
                }
            }
            m_last = dec.m;
            if constexpr (REC) {
                if (dec.accept && n_acc < p.rec_cap) {
                    // the step's start as the attempt used it: y_n, t_n and dt_n in float64 (t_n + dt_n is t1_acc), and f0
                    // when it is not a function of y_n (no FSAL: the previous step's last k)
                    const long long slot = n_acc * p.n_rows + r;
                    T *ry = (T *)p.rec_y + slot * D;
#pragma unroll
                    for (int d = 0; d < D; ++d) ry[d] = y[d];
                    if (!p.tab.fsal) {
                        T *rf = (T *)p.rec_f0 + slot * D;
#pragma unroll
                        for (int d = 0; d < D; ++d) rf[d] = f0[d];
                    }
                    p.rec_t[2 * slot] = t_cur;
                    p.rec_t[2 * slot + 1] = dt;
                }
            }
            if (dec.accept) {                                               // dopri5.py:113-120
                ++n_acc;
                t_cur = t1n;
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    y[d] = yi[d];
                    f0[d] = k[S - 1][d];
                }
            } else {
                ++n_rej;
            }
            cur = c_new;
            nadv = nadv2;
            dt = dec.dt_next;
            status = st_bits;
            done = dn;
        }
        p.n_acc[r] = n_acc;
        p.n_rej[r] = n_rej;
        p.dt_next[r] = dt;
        p.error_ratio[r] = m_last;
        p.status[r] = (int)status;
    }
}

// Launches the kernel instance K over `rows` rows on a grid whose blocks all stay resident, min(ceil(rows / threads), blocks
// per SM x SMs), timed and counted as the fused family.  K's occupancy (`name` in the refusal) and the SM count are queried
// once per process and device.
template <auto K, typename P>
static int launch_resident(const P &p, long long rows, int threads, const char *name, cudaStream_t st) {
    static std::mutex mu;
    static int per_sm[kFusedMaxDevices], nsm[kFusedMaxDevices];
    int dev = 0;
    B2_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= kFusedMaxDevices) return b2_fail(B2ODE_EINVAL, "device ordinal %d out of range", dev);
    int blocks_per_sm = 0, sms = 0;
    {
        std::lock_guard<std::mutex> lock(mu);
        if (per_sm[dev] == 0) {
            B2_CUDA(cudaDeviceGetAttribute(&nsm[dev], cudaDevAttrMultiProcessorCount, dev));
            B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm[dev], K, threads, 0));
            if (per_sm[dev] < 1) return b2_fail(B2ODE_ESTATE, "%s does not fit on an SM", name);
        }
        blocks_per_sm = per_sm[dev];
        sms = nsm[dev];
    }
    const long long need = (rows + threads - 1) / threads;
    const long long resident = (long long)blocks_per_sm * sms;
    const int grid = (int)(need < resident ? need : resident);
    const int slot = b2_timing_begin(6 /* B2_FAM_FUSED */, st);
    K<<<grid, threads, 0, st>>>(p);
    B2_CUDA(cudaGetLastError());
    b2_timing_end(6, slot, st);
    b2_count_launch();
    return 0;
}

template <typename T, bool REC>
static int rows_dispatch(const RowsParams &p, int rhs_kind, int n_k, cudaStream_t st) {
    return dispatch_rhs<T>(rhs_kind, [&](auto rhs) {
        return dispatch_nk("independent-rows solve", n_k, [&](auto s) {
            using RHS = decltype(rhs);
            constexpr int S = decltype(s)::value;
            return launch_resident<k_rows_adaptive<T, RHS, S, REC>>(p, p.n_rows, RowsShape<T, RHS, S>::threads, "k_rows_adaptive", st);
        });
    });
}

extern "C" size_t b2ode_rows_workspace_bytes(void) { return 256; }   // [row hand-out counter, 8 B][unused]

// b2ode_rows_solve and b2ode_rows_solve_record: rec NULL launches the plain kernel
static int rows_solve(const b2ode_adaptive_desc *desc, const b2ode_rows_desc *r, const b2ode_rows_record_desc *rec) {
    if (!desc || !r) return b2_fail(B2ODE_EINVAL, "null argument");
    if (!r->y0 || !r->out || !r->t_out || !r->n_acc || !r->n_rej || !r->dt_next || !r->error_ratio || !r->status ||
        !r->workspace)
        return b2_fail(B2ODE_EINVAL, "null buffer");
    if (desc->nseg != 1) return b2_fail(B2ODE_EINVAL, "independent-rows solve takes a single-tensor state");
    long long n_rows = 0;
    {
        const int rc = check_rhs(&r->rhs, desc->seg_len[0], &n_rows);
        if (rc) return rc;
    }
    if (desc->dense_kind != 0 || desc->controller != B2ODE_CTRL_REFERENCE)
        return b2_fail(B2ODE_EINVAL, "independent-rows solve supports the quartic dense output and the reference controller only");
    if (int rc = check_nk("independent-rows solve", desc->n_k)) return rc;
    if (desc->dtype != B2ODE_F64 && desc->dtype != B2ODE_F32) return b2_fail(B2ODE_EINVAL, "dtype must be 0 or 1");
    if (n_rows < 1) return b2_fail(B2ODE_EINVAL, "empty batch");
    if (r->n_out < 1) return b2_fail(B2ODE_EINVAL, "n_out must be at least 1");
    if (r->workspace_bytes < b2ode_rows_workspace_bytes()) return b2_fail(B2ODE_ENOMEM, "workspace too small");
    if ((uintptr_t)r->workspace & 15u) return b2_fail(B2ODE_EINVAL, "workspace must be 16-byte aligned");
    if (rec) {
        if (!rec->ckpt || !rec->sched || rec->capacity < 1)
            return b2_fail(B2ODE_EINVAL, "b2ode_rows_solve_record: ckpt, sched and a capacity >= 1 are required");
        if (!desc->fsal && !rec->ckpt_f0)
            return b2_fail(B2ODE_EINVAL, "b2ode_rows_solve_record: a tableau without FSAL needs ckpt_f0");
    }
    const int D = rhs_row_dim(r->rhs.kind);
    cudaStream_t st = (cudaStream_t)r->cuda_stream;
    RowsParams p;
    memset(&p, 0, sizeof(p));
    if (rec) {
        p.rec_y = rec->ckpt;
        p.rec_f0 = desc->fsal ? nullptr : rec->ckpt_f0;
        p.rec_t = rec->sched;
        p.rec_cap = rec->capacity;
    }
    p.y0 = r->y0;
    p.out = r->out;
    p.n_rows = n_rows;
    p.next = (unsigned long long *)r->workspace;
    p.n_acc = (long long *)r->n_acc;
    p.n_rej = (long long *)r->n_rej;
    p.dt_next = r->dt_next;
    p.error_ratio = r->error_ratio;
    p.status = (int *)r->status;
    p.have_first_step = (r->first_step == r->first_step) ? 1 : 0;
    p.t_start = r->t_start;
    p.first_step = r->first_step;
    fill_rhs(p, r->rhs);
    fill_tableau(p.tab, *desc);
    fill_ctrl(p.c, *desc);
    p.c.n_out = r->n_out;
    p.c.t_out = r->t_out;
    p.c.n_global[0] = D;
    B2_CUDA(cudaMemsetAsync(r->workspace, 0, sizeof(unsigned long long), st));
    if (rec) {
        if (desc->dtype == B2ODE_F64) return rows_dispatch<double, true>(p, r->rhs.kind, desc->n_k, st);
        return rows_dispatch<float, true>(p, r->rhs.kind, desc->n_k, st);
    }
    if (desc->dtype == B2ODE_F64) return rows_dispatch<double, false>(p, r->rhs.kind, desc->n_k, st);
    return rows_dispatch<float, false>(p, r->rhs.kind, desc->n_k, st);
}

extern "C" int b2ode_rows_solve(const b2ode_adaptive_desc *desc, const b2ode_rows_desc *r) { return rows_solve(desc, r, nullptr); }

extern "C" int b2ode_rows_solve_record(const b2ode_adaptive_desc *desc, const b2ode_rows_desc *r, const b2ode_rows_record_desc *rec) {
    if (!rec) return b2_fail(B2ODE_EINVAL, "b2ode_rows_solve_record: null record");
    return rows_solve(desc, r, rec);
}

// ================================================================================================
// independent rows, back-propagation through the accepted steps (odeint options={'independent_rows': True, 'backprop':
// True}; DESIGN.md §4.2(g)).  One thread per row walks that row's recorded steps (b2ode_rows_solve_record) in reverse with
// the reverse state in registers, restating backprop._Backward.run for one row -- b2ode_bp_rhs's stage recompute and
// vector-Jacobian products, b2ode_bp_dense's dense-output VJP, b2ode_bp_combine's reverse combines -- operation for
// operation, so a row's gradient equals the shared-step backward pass of that row solved alone, bit for bit:
//   1. the stage inputs Y_i = y_n + sum_j (dt beta_ij) k_j (zero coefficients dropped) and k_{i+1} = f(Y_i); f0 is an
//      evaluation at y_n (FSAL tableaus, and adaptive Heun's first step) or the recorded f0.  The last k is never needed.
//   2. the dense output's VJP of the outputs the step emitted, (t_n, t_n + dt_n] (recovered from the recorded t_n, dt_n
//      and the increasing output times), into g0, lambda and the masked k's;
//   3. adaptive Heun: the cotangent of the next step's f0 (carry) into this step's last k;
//   4. the reverse stage sweep, mu_{i+1} = dense + sum_{l > i} (dt beta_{l,i+1}) nu_l + (dt b_{i+1}) lambda and
//      nu_i = RHS::vjp(Y_i, mu_{i+1}) (the reverse-time system negates mu, as k_bp_rhs does);
//   5. lambda_n = g0 + (sum nu_i + xi_0 + lambda) with xi_0 = J(y_n)^T mu_0 when f0 is an evaluation at y_n.
// The built-ins are autonomous (RHS::kAutonomous): no stage time is recorded or needed.
//
// PAR (a built-in whose weights are all trainable, RHS::kParams): rows go to blocks statically (grid stride) and a block
// walks its rows' steps in block-uniform rounds -- round q is step n_acc - 1 - q of every row that has it; rows with fewer
// steps idle.  After each stage VJP the live rows' (y, g) are staged in shared memory and summed in fp64 by RHS's parameter
// hooks in k_bp_rhs's order; the block partials go to the workspace and the last block to arrive adds them in block order.  The sums depend on
// the batch and sm_count only.  Without parameters no barrier is needed and rows are handed out dynamically.
// ================================================================================================
constexpr int kRowsBpThreads = 128;

struct RowsBpParams {
    const void *ckpt, *ckpt_f0;
    const double *sched;
    const long long *n_acc;
    const double *t_out;
    const void *grad_out;
    void *grad_y0;
    long long n_rows;
    int n_out, fsal, n_params;
    unsigned long long *next;          // row hand-out counter (frozen parameters), zeroed before the launch
    unsigned *ticket;                  // last-block ticket (PAR), zero before and after the launch
    double *part, *param_grad;
    double time_sign;
    double rhs[8];
    const void *rhs_data;
    // the tableau rows k_rows_bp reads, without the Tableau block: the block's layout moves them and changes how ptxas
    // allocates k_rows_bp's registers
    double beta[B2ODE_MAXK][B2ODE_MAXK];
    double c_sol[B2ODE_MAXK], c_mid[B2ODE_MAXK];
};

template <typename T, typename RHS, int S, bool PAR>
__global__ void __launch_bounds__(kRowsBpThreads) k_rows_bp(const __grid_constant__ RowsBpParams p) {
    static_assert(RHS::kAutonomous, "k_rows_bp records no stage times: the right-hand side must not depend on t");
    static_assert(!PAR || RHS::kParams, "parameter sums need a right-hand side with trainable weights");
    using A = Ar<T>;
    constexpr int D = RHS::D;
    constexpr int NT = kRowsBpThreads;
    using PS = ParShape<T, RHS, NT, PAR>;
    __shared__ T sw[RHS::kSmem];
    __shared__ T tile[PS::tile];
    __shared__ bool on_s[PS::rows];
    __shared__ double red[PS::red];
    __shared__ unsigned long long rounds_s;
    stage_weights<T, RHS>(p.rhs, p.rhs_data, sw, NT);
    const bool neg = (T)p.time_sign < T(0);
    const long long N = p.n_rows * D;
    const T *ckpt = (const T *)p.ckpt, *ckpt_f0 = (const T *)p.ckpt_f0, *gout = (const T *)p.grad_out;
    const double *t_out = p.t_out;
    // lambda enters k_j with dt b_j: for FSAL y_{n+1} is the last stage input, whose row of beta is b (zero past S - 2)
    auto lam_coef = [&](int j) -> double { return p.fsal ? p.beta[S - 2][j] : p.c_sol[j]; };
    auto in_mask = [&](int j) -> bool { return j == 0 || j == S - 1 || p.c_mid[j] != 0.0; };
    // which nu_i exist (b2ode_bp_rhs is launched only with a cotangent): uniform over rows
    bool have[S - 1];
#pragma unroll
    for (int i = S - 2; i >= 0; --i) {
        const int j = i + 1;
        bool h = in_mask(j) || lam_coef(j) != 0.0;
#pragma unroll
        for (int l = j; l < S - 1; ++l) h = h || (have[l] && p.beta[l][j] != 0.0);
        have[i] = h;
    }
    double acc[PS::acc];
#pragma unroll
    for (int q = 0; q < PS::acc; ++q) acc[q] = 0.0;
    // one stage VJP's parameter cotangents over the block's rows (k_bp_rhs's tiles and order); every thread calls it
    auto par_sum = [&](bool on, const T(&Y)[D], const T(&g)[D]) {
        if constexpr (PAR) par_tiles<T, RHS, NT>(p.rhs, sw, tile, on_s, on, Y, g, acc);
    };
    // Y = y_n + sum_{j <= i} (dt beta_ij) k_j, zero coefficients dropped (k_bp_rhs's rebuild)
    auto stage_input = [&](int i, T dt, const T(&y)[D], const T(&k)[S - 1][D], T(&Y)[D]) {
        T a[D];
        bool any = false;
#pragma unroll
        for (int j = 0; j < S - 1; ++j) {
            if (j > i || p.beta[i][j] == 0.0) continue;
            const T c = A::mul(dt, (T)p.beta[i][j]);
#pragma unroll
            for (int d = 0; d < D; ++d) a[d] = any ? A::add(a[d], A::mul(c, k[j][d])) : A::mul(c, k[j][d]);
            any = true;
        }
#pragma unroll
        for (int d = 0; d < D; ++d) Y[d] = any ? A::add(y[d], a[d]) : y[d];
    };
    auto eval = [&](const T(&Y)[D], T(&k)[D]) {
        T dy[D];
        RHS::eval(p.rhs, sw, T(0), Y, dy);
#pragma unroll
        for (int d = 0; d < D; ++d) k[d] = neg ? -dy[d] : dy[d];
    };
    // nu = J(Y)^T g for the (negated in reverse time) cotangent g
    auto vjp = [&](const T(&Y)[D], T(&g)[D], T(&nu)[D]) {
        if (neg) {
#pragma unroll
            for (int d = 0; d < D; ++d) g[d] = -g[d];
        }
        T f[D];
        RHS::vjp(p.rhs, sw, T(0), Y, g, f, nu);
    };

    // one reverse step n of row r; `act` false (PAR only): the row has no step n, it only joins the block's barriers.
    // lam: the cotangent of y_{n+1} in, of y_n out; carry: adaptive Heun's cotangent of the next step's f0 (have_carry)
    auto reverse_step = [&](long long r, long long n, bool act, T(&lam)[D], T(&carry)[D], bool &have_carry, int &hi) {
        T y[D], k[S - 1][D];
        double t0d = 0.0, dtd = 0.0;
        const bool fresh0 = p.fsal || n == 0;
        if (act) {
            const long long slot = n * p.n_rows + r;
#pragma unroll
            for (int d = 0; d < D; ++d) y[d] = ckpt[slot * D + d];
            t0d = p.sched[2 * slot];
            dtd = p.sched[2 * slot + 1];
            // ---- recompute the stages ----
            if (fresh0) {
                eval(y, k[0]);
            } else {
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    const T f = ckpt_f0[slot * D + d];   // the forward's f0 holds f(-t, y) unsigned in reverse time
                    k[0][d] = neg ? -f : f;
                }
            }
#pragma unroll
            for (int i = 0; i < S - 2; ++i) {
                T Y[D];
                stage_input(i, (T)dtd, y, k, Y);
                eval(Y, k[i + 1]);
            }
        } else {
#pragma unroll
            for (int d = 0; d < D; ++d) y[d] = T(0);
#pragma unroll
            for (int j = 0; j < S - 1; ++j)
#pragma unroll
                for (int d = 0; d < D; ++d) k[j][d] = T(0);
        }
        const T dt = (T)dtd;
        // ---- dense output VJP: outputs j in [lo, hi) are those in (t_n, t_n + dt_n] ----
        T g0[D], gmid[D], gf0[D], gf1[D];
        if (act) {
            const double t1d = t0d + dtd;
            while (hi > 1 && t_out[hi - 1] > t1d) --hi;
            int lo = hi;
            while (lo > 1 && t_out[lo - 1] > t0d) --lo;
            const T t0 = (T)t0d, den = A::sub((T)t1d, t0);
#pragma unroll
            for (int d = 0; d < D; ++d) {
                T a1;
                bp_dense_quartic<T>([&](int j) { return gout[(long long)j * N + r * D + d]; }, lo, hi, t_out, t0, den, dt,
                                    g0[d], a1, gmid[d], gf0[d], gf1[d]);
                lam[d] = A::add(lam[d], a1);
            }
            hi = lo;
        }
        auto mu_dense = [&](int j, int d) -> T {
            T v = bp_dense_k<T>(j, S - 1, dt, p.c_mid[j], gmid[d], gf0[d], gf1[d]);
            if (j == S - 1 && have_carry) v = A::add(v, carry[d]);          // adaptive Heun (step None: coefficient 1)
            return v;
        };
        // ---- reverse stage sweep ----
        T nus[S - 1][D];
#pragma unroll
        for (int i = S - 2; i >= 0; --i) {
            if (!have[i]) continue;
            const int j = i + 1;
            T Y[D], g[D];
            if (act) {
                bool any = false;
#pragma unroll
                for (int l = j; l < S - 1; ++l) {
                    if (!have[l] || p.beta[l][j] == 0.0) continue;
                    const T c = A::mul(dt, (T)p.beta[l][j]);
#pragma unroll
                    for (int d = 0; d < D; ++d) g[d] = any ? A::add(g[d], A::mul(c, nus[l][d])) : A::mul(c, nus[l][d]);
                    any = true;
                }
                if (lam_coef(j) != 0.0) {
                    const T c = A::mul(dt, (T)lam_coef(j));
#pragma unroll
                    for (int d = 0; d < D; ++d) g[d] = any ? A::add(g[d], A::mul(c, lam[d])) : A::mul(c, lam[d]);
                    any = true;
                }
                if (in_mask(j)) {
#pragma unroll
                    for (int d = 0; d < D; ++d) g[d] = any ? A::add(mu_dense(j, d), g[d]) : mu_dense(j, d);
                }
                stage_input(i, dt, y, k, Y);
                vjp(Y, g, nus[i]);
            }
            par_sum(act, Y, g);
        }
        // ---- mu_0: the cotangent of f0 ----
        T g[D];
        bool xi0 = false;
        if (act) {
            bool any = false;
#pragma unroll
            for (int l = 0; l < S - 1; ++l) {
                if (!have[l] || p.beta[l][0] == 0.0) continue;
                const T c = A::mul(dt, (T)p.beta[l][0]);
#pragma unroll
                for (int d = 0; d < D; ++d) g[d] = any ? A::add(g[d], A::mul(c, nus[l][d])) : A::mul(c, nus[l][d]);
                any = true;
            }
            if (lam_coef(0) != 0.0) {
                const T c = A::mul(dt, (T)lam_coef(0));
#pragma unroll
                for (int d = 0; d < D; ++d) g[d] = any ? A::add(g[d], A::mul(c, lam[d])) : A::mul(c, lam[d]);
                any = true;
            }
#pragma unroll
            for (int d = 0; d < D; ++d) g[d] = any ? A::add(mu_dense(0, d), g[d]) : mu_dense(0, d);
            xi0 = fresh0;
        }
        T xi[D];
        // xi_0 = J(y_n)^T mu_0 when f0 is an evaluation at y_n: every step with FSAL, else the first step only -- which PAR
        // rows reach in different rounds, so every round joins the parameter sum's barriers
        if (xi0) vjp(y, g, xi);
        par_sum(xi0, y, g);
        if (act) {
            if (!fresh0) {
#pragma unroll
                for (int d = 0; d < D; ++d) carry[d] = g[d];
            }
            have_carry = !fresh0;
            // ---- lambda_n = g0 + (sum nu_i + xi_0 + lambda_{n+1}) ----
            T s[D];
            bool any = false;
#pragma unroll
            for (int i = 0; i < S - 1; ++i) {
                if (!have[i]) continue;
#pragma unroll
                for (int d = 0; d < D; ++d) s[d] = any ? A::add(s[d], nus[i][d]) : nus[i][d];
                any = true;
            }
            if (xi0) {
#pragma unroll
                for (int d = 0; d < D; ++d) s[d] = any ? A::add(s[d], xi[d]) : xi[d];
                any = true;
            }
#pragma unroll
            for (int d = 0; d < D; ++d) lam[d] = A::add(g0[d], any ? A::add(s[d], lam[d]) : lam[d]);
        }
    };

    auto finish_row = [&](long long r, const T(&lam)[D]) {
        // grad_y0 = lambda_0 + grad_out[0] (_OdeintBackprop.backward)
#pragma unroll
        for (int d = 0; d < D; ++d) ((T *)p.grad_y0)[r * D + d] = A::add(lam[d], gout[r * D + d]);
    };

    if constexpr (!PAR) {
        const long long nthr = (long long)gridDim.x * NT;
        for (long long r = (long long)blockIdx.x * NT + threadIdx.x; r < p.n_rows; r = nthr + (long long)atomicAdd(p.next, 1ull)) {
            T lam[D], carry[D];
#pragma unroll
            for (int d = 0; d < D; ++d) lam[d] = carry[d] = T(0);
            bool have_carry = false;
            int hi = p.n_out;
            for (long long n = p.n_acc[r] - 1; n >= 0; --n) reverse_step(r, n, true, lam, carry, have_carry, hi);
            finish_row(r, lam);
        }
    } else {
        const long long stride = (long long)gridDim.x * NT;
        for (long long b0 = (long long)blockIdx.x * NT; b0 < p.n_rows; b0 += stride) {
            const long long r = b0 + threadIdx.x;
            const long long steps = r < p.n_rows ? p.n_acc[r] : 0;
            if (threadIdx.x == 0) rounds_s = 0ull;
            __syncthreads();
            atomicMax(&rounds_s, (unsigned long long)steps);
            __syncthreads();
            const long long rounds = (long long)rounds_s;
            T lam[D], carry[D];
#pragma unroll
            for (int d = 0; d < D; ++d) lam[d] = carry[d] = T(0);
            bool have_carry = false;
            int hi = p.n_out;
            for (long long q = 0; q < rounds; ++q) {
                const long long n = steps - 1 - q;
                reverse_step(r, n, n >= 0, lam, carry, have_carry, hi);
            }
            if (r < p.n_rows) finish_row(r, lam);
            __syncthreads();      // rounds_s is rewritten for the next chunk
        }
        const int P = p.n_params;
        par_block_partial<RHS, NT>(p.rhs, acc, red, p.part + (size_t)blockIdx.x * P);
        par_last_block<NT>(p.ticket, p.part, P, [&](int q, double s) { p.param_grad[q] = s; });
    }
}

// PAR: a static grid of at most 8 blocks per SM (the parameter sums' order is fixed by the batch and sm_count)
static long long rows_bp_par_grid(long long rows, int sm_count) { return capped_grid(rows, kRowsBpThreads, 8, sm_count); }

template <typename T, typename RHS, int S, bool PAR>
static int rows_bp_launch(const RowsBpParams &p, int sm_count, cudaStream_t st) {
    if constexpr (!PAR) {
        return launch_resident<k_rows_bp<T, RHS, S, PAR>>(p, p.n_rows, kRowsBpThreads, "k_rows_bp", st);
    } else {
        const int slot = b2_timing_begin(6 /* B2_FAM_FUSED */, st);
        k_rows_bp<T, RHS, S, PAR><<<(int)rows_bp_par_grid(p.n_rows, sm_count), kRowsBpThreads, 0, st>>>(p);
        B2_CUDA(cudaGetLastError());
        b2_timing_end(6, slot, st);
        b2_count_launch();
        return 0;
    }
}

template <typename T>
static int rows_bp_dispatch(const RowsBpParams &p, int rhs_kind, int n_k, int sm_count, cudaStream_t st) {
    return dispatch_rhs<T>(rhs_kind, [&](auto rhs) {
        using RHS = decltype(rhs);
        return dispatch_nk("independent-rows backprop", n_k, [&](auto s) {
            constexpr int S = decltype(s)::value;
            if constexpr (RHS::kParams) {
                if (p.n_params > 0) return rows_bp_launch<T, RHS, S, true>(p, sm_count, st);
            }
            return rows_bp_launch<T, RHS, S, false>(p, sm_count, st);
        });
    });
}

static int check_rows_bp_params(const b2ode_rhs_desc *rhs, int64_t rows, int n_params) {
    if (!rhs) return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: null right-hand side");
    const int D = rhs_row_dim(rhs->kind);
    if (D < 0) return b2_fail(B2ODE_EINVAL, "unknown built-in right-hand side %d", rhs->kind);
    if (rows < 1) return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: empty batch");
    long long r2 = 0;
    if (int rc = check_rhs(rhs, (long long)rows * D, &r2)) return rc;
    const int P = rhs_n_weights(rhs);
    if (n_params != 0 && n_params != P)
        return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: n_params %d: right-hand side %d takes 0 (frozen) or %d", n_params, rhs->kind, P);
    return 0;
}

// [row hand-out counter 8 B | ticket 4 B | 4 B][PAR: grid x n_params doubles of block partials]
extern "C" size_t b2ode_rows_bp_workspace_bytes(const b2ode_rhs_desc *rhs, int64_t rows, int n_params, int sm_count) {
    if (check_rows_bp_params(rhs, rows, n_params)) return 0;
    return 16 + (n_params > 0 ? 8 * (size_t)rows_bp_par_grid(rows, sm_count) * (size_t)n_params : 0);
}

extern "C" int b2ode_rows_bp(const b2ode_adaptive_desc *desc, const b2ode_rows_bp_desc *d) {
    if (!desc || !d) return b2_fail(B2ODE_EINVAL, "null argument");
    if (desc->nseg != 1) return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: the state is a single tensor of whole rows");
    const int D = rhs_row_dim(d->rhs.kind);
    if (D < 0) return b2_fail(B2ODE_EINVAL, "unknown built-in right-hand side %d", d->rhs.kind);
    if (desc->seg_len[0] % D != 0) return b2_fail(B2ODE_EINVAL, "state length %lld is not a multiple of the row size %d",
                                                  (long long)desc->seg_len[0], D);
    const long long n_rows = desc->seg_len[0] / D;
    if (int rc = check_rows_bp_params(&d->rhs, n_rows, d->n_params)) return rc;
    if (desc->dtype != B2ODE_F64 && desc->dtype != B2ODE_F32) return b2_fail(B2ODE_EINVAL, "dtype must be 0 or 1");
    if (desc->dense_kind != 0)
        return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: the tableau needs the quartic dense output");
    if (int rc = check_nk("independent-rows backprop", desc->n_k)) return rc;
    if (d->n_out < 2) return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: n_out must be at least 2");
    if (!d->ckpt || !d->sched || !d->n_acc || !d->t_out || !d->grad_out || !d->grad_y0 || !d->workspace)
        return b2_fail(B2ODE_EINVAL, "null buffer");
    if (!desc->fsal && !d->ckpt_f0) return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: a tableau without FSAL needs ckpt_f0");
    if (d->capacity < 1) return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: capacity must be at least 1");
    if (d->n_params > 0 && !d->param_grad) return b2_fail(B2ODE_EINVAL, "b2ode_rows_bp: parameter sums need param_grad");
    const size_t need = b2ode_rows_bp_workspace_bytes(&d->rhs, n_rows, d->n_params, d->sm_count);
    if (d->workspace_bytes < need) return b2_fail(B2ODE_ENOMEM, "workspace too small: %zu < %zu", d->workspace_bytes, need);
    if ((uintptr_t)d->workspace & 15u) return b2_fail(B2ODE_EINVAL, "workspace must be 16-byte aligned");
    RowsBpParams p;
    memset(&p, 0, sizeof(p));
    p.ckpt = d->ckpt;
    p.ckpt_f0 = desc->fsal ? nullptr : d->ckpt_f0;
    p.sched = d->sched;
    p.n_acc = (const long long *)d->n_acc;
    p.t_out = d->t_out;
    p.grad_out = d->grad_out;
    p.grad_y0 = d->grad_y0;
    p.n_rows = n_rows;
    p.n_out = d->n_out;
    p.fsal = desc->fsal;
    p.n_params = d->n_params;
    p.next = (unsigned long long *)d->workspace;
    p.ticket = (unsigned *)((char *)d->workspace + 8);
    p.part = (double *)((char *)d->workspace + 16);
    p.param_grad = d->param_grad;
    fill_rhs(p, d->rhs);
    for (int i = 0; i < B2ODE_MAXK; ++i) {
        for (int j = 0; j < B2ODE_MAXK; ++j) p.beta[i][j] = desc->beta[i][j];
        p.c_sol[i] = desc->c_sol[i];
        p.c_mid[i] = desc->c_mid[i];
    }
    cudaStream_t st = (cudaStream_t)d->cuda_stream;
    B2_CUDA(cudaMemsetAsync(d->workspace, 0, 16, st));
    if (desc->dtype == B2ODE_F64) return rows_bp_dispatch<double>(p, d->rhs.kind, desc->n_k, d->sm_count, st);
    return rows_bp_dispatch<float>(p, d->rhs.kind, desc->n_k, d->sm_count, st);
}

// ================================================================================================
// independent rows, backward pass (DESIGN.md §4.2(e)): odeint_adjoint (tfdiffeq/adjoint.py:110-169) of every row of a
// built-in right-hand side on its own, as if the row had been passed to odeint_adjoint alone with fused_vjp.  A row's
// backward pass reads that row's forward solution and loss cotangent and nothing else, so one thread runs all of it -- every
// interval [t_i, t_{i-1}], every attempt, the dL/dt_i terms -- with the augmented state (y, adj_y, adj_t, adj_params) in
// registers.  adj_t and adj_params (the 0-dim zero: no trainable weights) have the zero derivative; they enter the error norm
// and the dense output as the stage kernels form them.  A second launch sums the time gradient over the rows.
//
// A sibling of k_rows_adaptive rather than a template over the row state: the forward kernel keeps its instantiations, and
// this one carries two k arrays and the per-interval loop, whose register needs differ (ptxas table in DESIGN.md).
// ================================================================================================
struct RowsAdjParams {
    const void *ans, *grad_out;        // (n_out, rows, D)
    void *grad_y0;                     // (rows, D)
    double *t_grad;                    // n_out
    const double *t_out;               // n_out forward output times
    int n_out;
    long long n_rows;
    unsigned long long *next;          // workspace: row hand-out counter, zeroed before the launch
    unsigned *ticket;                  // workspace: arrival counter of the time-gradient sums, zero between launches
    double *adj_t;                     // workspace: [rows] each row's final adj_t
    double *part;                      // workspace: [grid][n_out] block partials of the time gradient
    long long *n_acc, *n_rej;          // per row, summed over the intervals
    double *dt_next, *error_ratio;     // per row, after the last attempt of the last interval
    int *status;
    int have_first_step;
    double first_step;
    double time_sign;                  // of the backward solves: -1 when they run toward smaller t
    double rhs[8];
    const void *rhs_data;
    Tableau tab;
    CtrlParams c;                      // n_global = {D, D, 1, 1}: each component's norm is over its own elements
};

// dL/dt_i of one row: <f(t_i, y_i), g_i> (adjoint.py:133-136), products and sum in fp64 in element order, rounded once to
// the state dtype.  The backward kernel subtracts it from the row's adj_t and the time-gradient kernel sums it over the
// rows: both call this function, so the summed term is the subtracted one, bit for bit.
template <typename T, typename RHS>
__device__ __forceinline__ T rows_dldt(const double *prm, const T *sw, T t, const T (&y)[RHS::D], const T (&g)[RHS::D]) {
    T f[RHS::D];
    RHS::eval(prm, sw, t, y, f);
    double s = 0.0;
#pragma unroll
    for (int d = 0; d < RHS::D; ++d) s = __dadd_rn(s, __dmul_rn((double)f[d], (double)g[d]));
    return (T)s;
}

// sum_j (dt c_j) * 0 over the terms the stage kernels list for a row of coefficients (b2ode_adaptive_create): the nonzero
// c_j; a stage row without one keeps a single zero-weight term (`keep_one`), the midpoint row starts from +0.  The
// contribution of a zero derivative (adj_t, adj_params) to a stage input, error estimate or midpoint, signed zeros included.
// `dtk` carries the sign of the time direction, the zero none (see `rhs` in k_rows_adaptive).
template <typename T>
__device__ __forceinline__ T zero_combine(const double *c, int n, T dtk, bool keep_one) {
    T acc = T(0);
    bool first = true;
    for (int j = 0; j < n; ++j) {
        if (c[j] != 0.0 || (keep_one && first && j == n - 1)) {
            const T term = Ar<T>::mul(Ar<T>::mul(dtk, (T)c[j]), T(0));
            acc = first ? term : Ar<T>::add(acc, term);
            first = false;
        }
    }
    return acc;
}

template <typename T, typename RHS, int S>
__global__ void __launch_bounds__(RowsShape<T, RHS, S>::threads) k_rows_adjoint(const __grid_constant__ RowsAdjParams p) {
    using A = Ar<T>;
    constexpr int D = RHS::D;
    __shared__ T sw[RHS::kSmem];
    stage_weights<T, RHS>(p.rhs, p.rhs_data, sw, blockDim.x);
    const bool rev = (T)p.time_sign < T(0);
    // (f, g^T df/dy) at g = -a without the minus sign of the reverse-time wrapper; dt factors carry it (see k_rows_adaptive)
    auto aug = [&](T t, const T(&yy)[D], const T(&aa)[D], T(&fy)[D], T(&fa)[D]) {
        T g[D];
#pragma unroll
        for (int d = 0; d < D; ++d) g[d] = -aa[d];
        RHS::vjp(p.rhs, sw, rev ? -t : t, yy, g, fy, fa);
    };
    const int n_out = p.n_out;
    const long long N = p.n_rows * D;
    const T *ans = (const T *)p.ans, *gout = (const T *)p.grad_out;
    const T rtol = (T)p.tab.rtol0, atol = (T)p.tab.atol0;
    const long long nthr = (long long)gridDim.x * blockDim.x;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < p.n_rows;
         r = nthr + (long long)atomicAdd(p.next, 1ull)) {
        T a[D], at = T(0);                                                  // adjoint.py:110-116
#pragma unroll
        for (int d = 0; d < D; ++d) a[d] = gout[(long long)(n_out - 1) * N + r * D + d];
        unsigned status = 0u;
        long long n_acc = 0, n_rej = 0;
        double dt = 0.0, m_last = 0.0;
        for (int i = n_out - 1; i >= 1 && status == 0u; --i) {             // adjoint.py:118
            T y[D];
            {
                T g[D];
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    y[d] = ans[(long long)i * N + r * D + d];
                    g[d] = gout[(long long)i * N + r * D + d];
                }
                at = A::sub(at, rows_dldt<T, RHS>(p.rhs, sw, (T)p.t_out[i], y, g));   // adjoint.py:138
            }
            // odeint(augmented_dynamics, (y_i, adj_y, adj_t, 0), [t_i, t_{i-1}]) in the time of the backward solve
            double t_cur = rev ? -p.t_out[i] : p.t_out[i];
            const double t_end = rev ? -p.t_out[i - 1] : p.t_out[i - 1];
            T fy[D], fa[D];
            aug((T)t_cur, y, a, fy, fa);
            if (p.have_first_step) {
                dt = p.first_step;
            } else {
                // _select_initial_step (misc.py:183-247), one norm per component, as k_init_norms / k_init_finish form them
                T sy[D], sa[D];
                Partial tot[4];
                double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    sy[d] = A::add(atol, A::mul(A::abs(y[d]), rtol));
                    sa[d] = A::add(atol, A::mul(A::abs(a[d]), rtol));
                    const double q0 = (double)A::div(y[d], sy[d]), q1 = (double)A::div(fy[d], sy[d]);
                    const double q2 = (double)A::div(a[d], sa[d]), q3 = (double)A::div(fa[d], sa[d]);
                    s0 += q0 * q0;
                    s1 += q1 * q1;
                    s2 += q2 * q2;
                    s3 += q3 * q3;
                }
                const T st = A::add(atol, A::mul(A::abs(at), rtol)), sp = A::add(atol, A::mul(T(0), rtol));
                const double qt = (double)A::div(at, st), qt1 = (double)A::div(T(0), st), qp = (double)A::div(T(0), sp);
                tot[0].v[0] = s0;
                tot[0].v[1] = s1;
                tot[1].v[0] = s2;
                tot[1].v[1] = s3;
                tot[2].v[0] = qt * qt;
                tot[2].v[1] = qt1 * qt1;
                tot[3].v[0] = tot[3].v[1] = qp * qp;
#pragma unroll
                for (int s = 0; s < 4; ++s) tot[s].v[2] = tot[s].v[3] = 0.0;
                T d1max;
                const T h0 = init_h0<T>(p.c, tot, 4, &d1max), hk = negate_if(h0, rev);
                T y1[D], a1[D], gy1[D], ga1[D];
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    y1[d] = A::add(y[d], A::mul(hk, fy[d]));
                    a1[d] = A::add(a[d], A::mul(hk, fa[d]));
                }
                aug(A::add((T)t_cur, h0), y1, a1, gy1, ga1);
                s0 = s2 = 0.0;
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    const double q0 = (double)A::div(A::sub(gy1[d], fy[d]), sy[d]);
                    const double q2 = (double)A::div(A::sub(ga1[d], fa[d]), sa[d]);
                    s0 += q0 * q0;
                    s2 += q2 * q2;
                }
                tot[0].v[0] = s0;
                tot[1].v[0] = s2;
                tot[2].v[0] = qt1 * qt1;                                    // (0 - 0) / scale
                tot[3].v[0] = qp * qp;
                dt = (double)init_dt<T>(p.c, tot, 4, h0, d1max);
            }
            T aout[D], atout = at;
            bool done = false;
            if (step_underflows(t_cur, dt)) {
                status |= B2ODE_ST_UNDERFLOW;
                done = true;
            }
            long long nadv = 0;
            while (!done) {
                const T t0c = (T)t_cur, dtc = (T)dt;
                const T dtk = negate_if(dtc, rev);
                T k[S][D], ka[S][D], yi[D], ai[D];
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    k[0][d] = fy[d];
                    ka[0][d] = fa[d];
                }
#pragma unroll
                for (int s = 0; s < S - 1; ++s) {
                    const T ti = A::add(t0c, A::mul((T)p.c.alpha[s], dtc));
                    T ay[D], aa[D];
#pragma unroll
                    for (int j = 0; j <= s; ++j) {
                        const T c = A::mul(dtk, (T)p.tab.beta[s][j]);
#pragma unroll
                        for (int d = 0; d < D; ++d) {
                            const T ty = A::mul(c, k[j][d]), ta = A::mul(c, ka[j][d]);
                            ay[d] = (j == 0) ? ty : A::add(ay[d], ty);
                            aa[d] = (j == 0) ? ta : A::add(aa[d], ta);
                        }
                    }
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        yi[d] = A::add(y[d], ay[d]);
                        ai[d] = A::add(a[d], aa[d]);
                    }
                    aug(ti, yi, ai, k[s + 1], ka[s + 1]);
                }
                if (!p.tab.fsal) {
                    T ay[D], aa[D];
#pragma unroll
                    for (int j = 0; j < S; ++j) {
                        const T c = A::mul(dtk, (T)p.tab.c_sol[j]);
#pragma unroll
                        for (int d = 0; d < D; ++d) {
                            const T ty = A::mul(c, k[j][d]), ta = A::mul(c, ka[j][d]);
                            ay[d] = (j == 0) ? ty : A::add(ay[d], ty);
                            aa[d] = (j == 0) ? ta : A::add(aa[d], ta);
                        }
                    }
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        yi[d] = A::add(y[d], ay[d]);
                        ai[d] = A::add(a[d], aa[d]);
                    }
                }
                // adj_t at the end of the attempt: the last stage row (FSAL; adaptive_heun's only row is stage 0's single
                // term) or the solution row, over a zero derivative
                const T at1 = A::add(at, p.tab.fsal ? zero_combine<T>(p.tab.beta[S - 2], S - 1, dtk, true)
                                                : zero_combine<T>(p.tab.c_sol, S, dtk, true));
                // error estimate and norm terms of y and adj_y in element order (norm_terms' operations); adj_t's error is a
                // zero, adj_params is the zero
                Partial tot[4];
                {
                    double sy = 0.0, sa = 0.0;
                    unsigned long long m0 = 0ull, m1 = 0ull, n0 = 0ull, n1 = 0ull;
                    T ey[D], ea[D];
#pragma unroll
                    for (int j = 0; j < S; ++j) {
                        const T c = A::mul(dtk, (T)p.tab.c_error[j]);
#pragma unroll
                        for (int d = 0; d < D; ++d) {
                            const T ty = A::mul(c, k[j][d]), ta = A::mul(c, ka[j][d]);
                            ey[d] = (j == 0) ? ty : A::add(ey[d], ty);
                            ea[d] = (j == 0) ? ta : A::add(ea[d], ta);
                        }
                    }
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        sy += (double)ey[d] * (double)ey[d];
                        sa += (double)ea[d] * (double)ea[d];
                        m0 = umax64(m0, (unsigned long long)__double_as_longlong(fabs((double)y[d])));
                        m1 = umax64(m1, (unsigned long long)__double_as_longlong(fabs((double)yi[d])));
                        n0 = umax64(n0, (unsigned long long)__double_as_longlong(fabs((double)a[d])));
                        n1 = umax64(n1, (unsigned long long)__double_as_longlong(fabs((double)ai[d])));
                    }
                    tot[0].v[0] = sy;
                    tot[0].v[1] = tot[0].v[2] = __longlong_as_double((long long)umax64(m0, m1));
                    tot[0].v[3] = (m0 >= 0x7ff0000000000000ull) ? 1.0 : 0.0;
                    tot[1].v[0] = sa;
                    tot[1].v[1] = tot[1].v[2] = __longlong_as_double((long long)umax64(n0, n1));
                    tot[1].v[3] = (n0 >= 0x7ff0000000000000ull) ? 1.0 : 0.0;
                    tot[2].v[0] = 0.0;
                    tot[2].v[1] = fabs((double)at);
                    tot[2].v[2] = fabs((double)at1);
                    tot[2].v[3] = isfinite((double)at) ? 0.0 : 1.0;
                    tot[3].v[0] = tot[3].v[1] = tot[3].v[2] = tot[3].v[3] = 0.0;
                }
                // the fp64 products above are the stage kernels' `ed * ed`; ctrl_decide as in k_rk_finalize, four components
                const CtrlDecision dec = ctrl_decide<T>(p.c, tot, 4, dt);
                const double t1_acc = t_cur + dt;
                // advance() over the one output time t_{i-1}: cursor 1 of the outputs (t_i, t_{i-1})
                const StepAdvance nx = advance_step(dec, status, 1, t_end <= t1_acc ? 2 : 1, 2, nadv, p.c.max_num_steps, t_cur, dt);
                if (nx.cur > 1) {
                    // dense output at t_{i-1} of adj_y and adj_t (y restarts from the forward solution): quartic_fit, quartic_eval
                    const DenseConst<T, S> dc = dense_const<T, S>(p.tab, dtk);
                    const T t0s = t0c, den = A::sub((T)t1_acc, t0s);
                    const T x = A::div(A::sub((T)t_end, t0s), den);
                    const T x2 = A::mul(x, x), x3 = A::mul(x2, x), x4 = A::mul(x3, x);
                    auto fit = [&](T f0e, T f1e, T y0e, T y1e, T ymd) {
                        T ca, cb, cc, cd;
                        quartic_fit<T, S>(dc, dtk, f0e, f1e, y0e, y1e, ymd, ca, cb, cc, cd);
                        return quartic_eval<T>(ca, cb, cc, cd, y0e, x, x2, x3, x4);
                    };
                    {
                        T ymid[1][D];
                        tableau_combine<T>(ymid, S, [&](int j) { return dc.cmid[j]; }, [&](int j, int, int d) { return ka[j][d]; });
#pragma unroll
                        for (int d = 0; d < D; ++d) aout[d] = fit(ka[0][d], ka[S - 1][d], a[d], ai[d], A::add(a[d], ymid[0][d]));
                    }
                    atout = fit(T(0), T(0), at, at1, A::add(at, zero_combine<T>(p.tab.c_mid, S, dtk, false)));
                }
                m_last = dec.m;
                if (dec.accept) {                                           // dopri5.py:113-120
                    ++n_acc;
                    t_cur = nx.t1;
                    at = at1;
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        y[d] = yi[d];
                        a[d] = ai[d];
                        fy[d] = k[S - 1][d];
                        fa[d] = ka[S - 1][d];
                    }
                } else {
                    ++n_rej;
                }
                nadv = nx.nadv;
                dt = dec.dt_next;
                status = nx.status;
                done = nx.done;
            }
            if (status == 0u) {
#pragma unroll
                for (int d = 0; d < D; ++d) a[d] = A::add(aout[d], gout[(long long)(i - 1) * N + r * D + d]);   // adjoint.py:164
                at = atout;
            }
        }
        T *gy0 = (T *)p.grad_y0;
#pragma unroll
        for (int d = 0; d < D; ++d) gy0[r * D + d] = a[d];
        p.adj_t[r] = (double)at;
        p.n_acc[r] = n_acc;
        p.n_rej[r] = n_rej;
        p.dt_next[r] = dt;
        p.error_ratio[r] = m_last;
        p.status[r] = (int)status;
    }
}

// t_grad[i] = sum over rows of dL/dt_{r,i} (i >= 1) and t_grad[0] = sum over rows of the final adj_t (adjoint.py:168-169).
// Rows are assigned to blocks statically (grid stride), each block sums its rows in fp64 in a fixed order into one partial
// per output time, and the last block to arrive adds the partials in block order: the sums depend on the grid -- a function
// of the batch and the SM count -- but not on timing or on the backward kernel's row hand-out.  No (n_out x rows) buffer.
template <typename T, typename RHS>
__global__ void __launch_bounds__(kThreads) k_rows_adjoint_tgrad(const __grid_constant__ RowsAdjParams p) {
    constexpr int D = RHS::D;
    __shared__ T sw[RHS::kSmem];
    stage_weights<T, RHS>(p.rhs, p.rhs_data, sw, kThreads);
    const long long N = p.n_rows * D;
    const long long stride = (long long)gridDim.x * kThreads;
    const T *ans = (const T *)p.ans, *gout = (const T *)p.grad_out;
    for (int i = 0; i < p.n_out; ++i) {
        double s = 0.0;
        for (long long r = (long long)blockIdx.x * kThreads + threadIdx.x; r < p.n_rows; r += stride) {
            if (i == 0) {
                s += p.adj_t[r];
            } else {
                T y[D], g[D];
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    y[d] = ans[(long long)i * N + r * D + d];
                    g[d] = gout[(long long)i * N + r * D + d];
                }
                s += (double)rows_dldt<T, RHS>(p.rhs, sw, (T)p.t_out[i], y, g);
            }
        }
        Partial x;
        x.v[0] = s;
        x.v[1] = x.v[2] = x.v[3] = 0.0;
        const Partial b = block_reduce<0u>(x);
        if (threadIdx.x == 0) p.part[(size_t)blockIdx.x * p.n_out + i] = b.v[0];
    }
    if (!last_block_arrives(p.ticket)) return;
    for (int i = threadIdx.x; i < p.n_out; i += kThreads) {
        double s = 0.0;
        for (unsigned b = 0; b < gridDim.x; ++b) s += __ldcg(p.part + (size_t)b * p.n_out + i);
        p.t_grad[i] = s;
    }
    if (threadIdx.x == 0) *p.ticket = 0;
}

static long long rows_adjoint_tgrad_grid(long long rows, int sm_count) { return capped_grid(rows, kThreads, 2, sm_count); }

template <typename T, typename RHS, int S>
static int rows_adjoint_launch(const RowsAdjParams &p, int sm_count, cudaStream_t st) {
    if (int rc = launch_resident<k_rows_adjoint<T, RHS, S>>(p, p.n_rows, RowsShape<T, RHS, S>::threads, "k_rows_adjoint", st))
        return rc;
    k_rows_adjoint_tgrad<T, RHS><<<(int)rows_adjoint_tgrad_grid(p.n_rows, sm_count), kThreads, 0, st>>>(p);
    B2_CUDA(cudaGetLastError());
    b2_count_launch();
    return 0;
}

template <typename T>
static int rows_adjoint_dispatch(const RowsAdjParams &p, int rhs_kind, int n_k, int sm_count, cudaStream_t st) {
    return dispatch_rhs<T>(rhs_kind, [&](auto rhs) {
        return dispatch_nk("independent-rows backward pass", n_k,
                           [&](auto s) { return rows_adjoint_launch<T, decltype(rhs), decltype(s)::value>(p, sm_count, st); });
    });
}

// [row hand-out counter 8 B | ticket 4 B | 4 B][adj_t: rows doubles][partials: grid x n_out doubles]
extern "C" size_t b2ode_rows_adjoint_workspace_bytes(int64_t rows, int32_t n_out, int sm_count) {
    if (rows < 1 || n_out < 1) return 0;
    return 16 + 8 * (size_t)rows + 8 * (size_t)rows_adjoint_tgrad_grid(rows, sm_count) * (size_t)n_out;
}

extern "C" int b2ode_rows_adjoint_solve(const b2ode_adaptive_desc *desc, const b2ode_rows_adjoint_desc *r) {
    if (!desc || !r) return b2_fail(B2ODE_EINVAL, "null argument");
    long long n_rows = 0;
    {
        int P = 0;
        const int rc = check_adjoint_rhs(&r->rhs, desc->nseg, desc->seg_len, &n_rows, &P);
        if (rc) return rc;
        if (P != 0)
            return b2_fail(B2ODE_EINVAL, "independent-rows backward pass takes frozen weights only (adj_params of 1 element)");
    }
    if (!r->ans || !r->grad_out || !r->t_out || !r->grad_y0 || !r->t_grad || !r->n_acc || !r->n_rej || !r->dt_next ||
        !r->error_ratio || !r->status || !r->workspace)
        return b2_fail(B2ODE_EINVAL, "null buffer");
    if (desc->dense_kind != 0 || desc->controller != B2ODE_CTRL_REFERENCE)
        return b2_fail(B2ODE_EINVAL, "independent-rows backward pass supports the quartic dense output and the reference controller only");
    if (int rc = check_nk("independent-rows backward pass", desc->n_k)) return rc;
    if (desc->dtype != B2ODE_F64 && desc->dtype != B2ODE_F32) return b2_fail(B2ODE_EINVAL, "dtype must be 0 or 1");
    if (r->n_out < 2) return b2_fail(B2ODE_EINVAL, "n_out must be at least 2 (one backward interval)");
    const size_t need = b2ode_rows_adjoint_workspace_bytes(n_rows, r->n_out, desc->sm_count);
    if (r->workspace_bytes < need) return b2_fail(B2ODE_ENOMEM, "workspace too small: %zu < %zu", r->workspace_bytes, need);
    if ((uintptr_t)r->workspace & 15u) return b2_fail(B2ODE_EINVAL, "workspace must be 16-byte aligned");
    const int D = rhs_row_dim(r->rhs.kind);
    cudaStream_t st = (cudaStream_t)r->cuda_stream;
    RowsAdjParams p;
    memset(&p, 0, sizeof(p));
    p.ans = r->ans;
    p.grad_out = r->grad_out;
    p.grad_y0 = r->grad_y0;
    p.t_grad = r->t_grad;
    p.t_out = r->t_out;
    p.n_out = r->n_out;
    p.n_rows = n_rows;
    p.next = (unsigned long long *)r->workspace;
    p.ticket = (unsigned *)((char *)r->workspace + 8);
    p.adj_t = (double *)((char *)r->workspace + 16);
    p.part = p.adj_t + n_rows;
    p.n_acc = (long long *)r->n_acc;
    p.n_rej = (long long *)r->n_rej;
    p.dt_next = r->dt_next;
    p.error_ratio = r->error_ratio;
    p.status = (int *)r->status;
    p.have_first_step = (r->first_step == r->first_step) ? 1 : 0;
    p.first_step = r->first_step;
    fill_rhs(p, r->rhs);
    fill_tableau(p.tab, *desc);
    fill_ctrl(p.c, *desc);
    p.c.n_out = 2;
    p.c.n_global[0] = p.c.n_global[1] = D;
    p.c.n_global[2] = p.c.n_global[3] = 1;
    B2_CUDA(cudaMemsetAsync(r->workspace, 0, 16, st));
    if (desc->dtype == B2ODE_F64) return rows_adjoint_dispatch<double>(p, r->rhs.kind, desc->n_k, desc->sm_count, st);
    return rows_adjoint_dispatch<float>(p, r->rhs.kind, desc->n_k, desc->sm_count, st);
}
