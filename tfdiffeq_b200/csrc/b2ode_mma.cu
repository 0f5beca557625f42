// b2ode_mma.cu -- the GEMM-shaped part of the path: a dense layer of an ODENet-style func on Hopper's tensor cores.
//
// SURVEY.md 8(f)-3 / north_star: "tensor cores used only when func is the ODENet linear block (a genuine dense
// GEMM)".  The reference's ODEFunc is fc1 -> relu -> fc2 -> relu -> fc3 (tfdiffeq/models/dense_odenet.py:85-92).
// One kernel computes   out[M, N] = act( A[M, K] . W[N, K]^T + bias[N] )   with fp32 storage and TF32 tensor-core
// math (TensorFlow's own default for fp32 matmuls on Ampere and later), where A is either a plain activation
// matrix or -- for the first layer -- the Runge-Kutta stage input produced on the fly,
//     A = y0 + sum_j (dt * beta_j) * k_j          (tfdiffeq/rk_common.py:51, dt read from the device state),
// i.e. the stage combine is the A-operand producer and the stage input never round-trips HBM for the GEMM.
//
// Hopper (sm_90a) mapping: one CTA of two warpgroups per 128-row tile, each warpgroup owning 64 rows; operands are
// written by the threads themselves into the canonical K-major SWIZZLE_128B shared-memory layout (they are computed,
// not copied, so there is nothing for TMA to fetch); wgmma.mma_async m64n64k8 TF32 instructions read both operands
// from shared memory through matrix descriptors and accumulate in fp32 registers; the epilogue adds the bias, applies
// the activation and stores fp32 rows straight from the accumulator fragments.

#include "b2ode_dev.cuh"

#include <stdint.h>
#include <stdlib.h>

constexpr int kTileM = 128;
constexpr int kKChunk = 64;              // K elements staged per round: 2 swizzle blocks of 32 tf32 (128 bytes)
constexpr int kMaxNK = 8;
constexpr int kWgThreads = 128;          // one warpgroup: the unit that issues a wgmma
constexpr int kConsumerThreads = 2 * kWgThreads;   // two warpgroups x 64 rows = one 128-row tile
constexpr int kNSub = 64;                // output columns per wgmma (m64n64k8); a tile of N columns issues ceil(N / 64)

struct DenseParams {
    const float *x;                      // A (nk == 0) or y0 (nk > 0), row-major [M, K]
    const float *k[kMaxNK];              // stage derivatives, row-major [M, K]
    double coef[kMaxNK];                 // beta_j of the stage row (zeros already dropped)
    int nk;
    const b2ode_state *st;               // dt lives here when nk > 0
    float *ystage;                       // optional: also materialise the stage input (needed for the last stage)
    const float *W;                      // [N, K] row-major (torch nn.Linear.weight layout), values already rounded to TF32
    const float *W_lo;                   // null: plain TF32.  Else tf32(W_fp32 - W): the 3xTF32 split (fp32-accurate products)
    const float *bias;                   // [N] or null
    float *out;                          // [M, N]
    int M, K, N;
    int act;                             // 0 none, 1 relu, 2 tanh, 3 softplus
    // 16-byte loads / stores (else element by element), decided by the host per operand group: A (x, every k[j],
    // ystage) when K % 4 == 0 and all of them are 16-byte aligned, B (W, W_lo) likewise
    int vec_a, vec_w;
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint32_t to_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}

// low half of the 3xTF32 split: tf32(x - tf32(x)); the subtraction is exact in fp32
__device__ __forceinline__ uint32_t tf32_lo(float x) {
    return to_tf32(__fsub_rn(x, __uint_as_float(to_tf32(x))));
}

// Round to TF32's 11 significant bits with three FP32 operations (Veltkamp's split, C = 2^13 + 1): round-to-nearest
// (ties to even), low 13 mantissa bits come out zero, NaN and Inf stay non-finite.  cvt.rna.tf32.f32 has no fast
// hardware path (ptxas emulates it in several integer/predicate instructions); this is what the activation epilogues use.
// |x| > 4e34 overflows the intermediate product and yields NaN.
__device__ __forceinline__ uint32_t to_tf32_fast(float x) {
    const float g = __fmul_rn(x, 8193.0f);
    const float d = __fsub_rn(x, g);
    return __float_as_uint(__fadd_rn(g, d));
}

// byte offset of (row, 16-byte chunk c in 0..7) inside one [rows x 128 B] K-major SWIZZLE_128B block:
// 8-row atoms of 1024 B, the chunk index XOR-ed with the row inside the atom (Swizzle<3,4,3>)
__device__ __forceinline__ uint32_t sw128_offset(int row, int chunk) {
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((chunk ^ (row & 7)) << 4));
}

// ---- wgmma plumbing ----------------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (sm_90), K-major SWIZZLE_128B: start address >> 4 in bits [0,14), leading byte offset
// (unused for swizzled K-major, 1) in [16,30), stride byte offset 1024 >> 4 (dense 8-row atoms) in [32,46), layout type 1
// (128-byte swizzle) in [62,64).  The high word is a constant; the low word is (address >> 4) | LBO, so a K step of
// 8 TF32 (32 bytes) inside the swizzle atom is `+ 2` and the next 8-row atom is `+ 64`.  Every operand base is
// 1024-byte aligned, so the descriptor's base-offset field stays 0.
constexpr uint32_t kDescHi = (uint32_t)(1024 >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr) { return ((saddr & 0x3FFFF) >> 4) | (1u << 16); }
__device__ __forceinline__ uint64_t desc(uint32_t lo) { return ((uint64_t)kDescHi << 32) | (uint64_t)lo; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Pins accumulator registers in place around the asynchronous MMAs: without it the compiler may read (or move) an
// accumulator between the wgmma that writes it and the wgmma.wait_group that makes the value valid.
template <int NS>
__device__ __forceinline__ void fence_acc(float (&acc)[4][32]) {
#pragma unroll
    for (int j = 0; j < NS; ++j)
#pragma unroll
        for (int r = 0; r < 32; ++r) asm volatile("" : "+f"(acc[j][r])::"memory");
}

// D[64 x 64] (+)= A[64 x 8] . B[64 x 8]^T, TF32 operands from shared memory, fp32 accumulators in registers.
// Fragment layout of D: warp w of the warpgroup holds rows 16w .. 16w + 15; register 4q + 2i + c of lane l is
// (row 16w + l / 4 + 8i, column 8q + 2 (l % 4) + c).
__device__ __forceinline__ void wgmma_m64n64k8_tf32(float (&d)[32], uint64_t da, uint64_t db, uint32_t accum) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accum));
}

// One 32-column K block (four K steps of 8) of a 64 x (64 NS) product: A at a_lo (64 rows), B at b_lo (64 NS rows)
template <int NS>
__device__ __forceinline__ void mma_kblock(float (&acc)[4][32], uint32_t a_lo, uint32_t b_lo, bool accum_first) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int j = 0; j < NS; ++j)
            wgmma_m64n64k8_tf32(acc[j], desc(a_lo + 2u * ks), desc(b_lo + (uint32_t)j * ((kNSub * 128) >> 4) + 2u * ks),
                                (ks > 0 || accum_first) ? 1u : 0u);
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}

// barrier over the threads of the two consumer warpgroups only (the chained kernel's loader warp does not take part)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory"); }
__device__ __forceinline__ void warpgroup_sync(int wg) { asm volatile("bar.sync %0, %1;" ::"r"(2 + wg), "n"(kWgThreads) : "memory"); }

// compile-time activation: a run-time switch inlined per element bloats the unrolled epilogues past the
// instruction cache (tanhf + log1pf/expf bodies many times over) even when only the relu branch ever executes
template <int ACT>
__device__ __forceinline__ float act_t(float v) {
    if (ACT == 1) return v > 0.f ? v : 0.f;
    if (ACT == 2) return tanhf(v);
    if (ACT == 3) return (v > 20.f) ? v : log1pf(expf(v));
    return v;
}

// ---- operand producers (shared by the dense-layer kernel and the chained kernel) ----------------------------------
// Fill one K chunk (64 columns) of the B operand (NT rows of W, host-rounded TF32) and of the A operand (128 rows:
// a plain activation tile, or the Runge-Kutta stage input formed on the fly) in the K-major SWIZZLE_128B layout.
// Called by NTHR threads with ids 0..NTHR-1.  NK (the number of k's in the stage combine) is a template parameter
// so that every global load of a batch -- BQ positions x (1 + NK) streams -- is issued before the first one is
// consumed: the producers are latency-bound, memory-level parallelism is what feeds the tensor core.
// 3xTF32 (p.W_lo != null): every fp32 operand is split as x = hi + lo with hi = tf32(x), lo = tf32(x - hi), and the
// product is accumulated in fp32 (registers) as A_lo.W_hi + A_hi.W_lo + A_hi.W_hi -- the K loop simply runs three times
// over the same columns with `mode` selecting which halves are staged (1: A_lo/W_hi, 2: A_hi/W_lo, 0: A_hi/W_hi).
// The dropped A_lo.W_lo term is 2^-22 relative: the result is as accurate as an fp32 FMA chain.
template <int NTHR, int NK>
__device__ __forceinline__ void produce_chunk_t(const DenseParams &p, uint8_t *sA, uint8_t *sB, int m0, int n0, int NT, int kc,
                                                int tid, const float (&cf)[kMaxNK], int mode) {
    const float *Wsrc = (mode == 2) ? p.W_lo : p.W;
    // ---- B chunk first: NT rows (output features) x 64 columns of W[N, K], already TF32-rounded by the host:
    //      raw 16-byte async copies straight into the swizzled layout (no register staging), zero-filled past K
    if (p.vec_w) {
        for (int f = tid; f < NT * (kKChunk / 4); f += NTHR) {
            const int row = f / (kKChunk / 4), c4 = f % (kKChunk / 4);
            const int gk = kc + c4 * 4;
            const float *src = Wsrc + (size_t)(n0 + row) * p.K + (gk < p.K ? gk : 0);
            const uint32_t dst = smem_u32(sB + (c4 >> 3) * (256 * 128) + sw128_offset(row, c4 & 7));
            const int nbytes = gk < p.K ? 16 : 0;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(nbytes) : "memory");
        }
    } else {
        for (int f = tid; f < NT * (kKChunk / 4); f += NTHR) {
            const int row = f / (kKChunk / 4), c4 = f % (kKChunk / 4);
            const int gk = kc + c4 * 4;
            uint32_t e[4] = {0u, 0u, 0u, 0u};
            for (int q = 0; q < 4 && gk + q < p.K; ++q) e[q] = __float_as_uint(Wsrc[(size_t)(n0 + row) * p.K + gk + q]);
            *reinterpret_cast<uint4 *>(sB + (c4 >> 3) * (256 * 128) + sw128_offset(row, c4 & 7)) = make_uint4(e[0], e[1], e[2], e[3]);
        }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    // ---- A chunk: 128 rows x 64 columns = PP float4 per thread
    constexpr int PP = kTileM * (kKChunk / 4) / NTHR;          // 8 float4 per thread (256 threads)
    // positions per batch: (1 + NK) x BQ float4 live at once, next to the 128 accumulator registers of an in-flight GEMM
    constexpr int BQ = (NK == 0) ? PP : (NK >= 4 ? 2 : 4);
    if (p.vec_a) {
#pragma unroll 1
        for (int b0 = 0; b0 < PP; b0 += BQ) {
            float4 v[BQ];
            float4 kv[NK > 0 ? NK : 1][BQ];
            size_t off[BQ];
            bool in[BQ];
#pragma unroll
            for (int q = 0; q < BQ; ++q) {
                const int f = tid + (b0 + q) * NTHR;
                const int row = f / (kKChunk / 4), c4 = f % (kKChunk / 4);
                const int gm = m0 + row, gk = kc + c4 * 4;
                in[q] = gm < p.M && gk < p.K;
                off[q] = in[q] ? (size_t)gm * p.K + gk : 0;
            }
            // all loads of the batch first ...
#pragma unroll
            for (int q = 0; q < BQ; ++q)
                v[q] = in[q] ? *reinterpret_cast<const float4 *>(p.x + off[q]) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int j = 0; j < NK; ++j)
#pragma unroll
                for (int q = 0; q < BQ; ++q)
                    kv[j][q] = in[q] ? *reinterpret_cast<const float4 *>(p.k[j] + off[q]) : make_float4(0.f, 0.f, 0.f, 0.f);
            // ... then the combine (rk_common.py:51: (dt*beta_j)*k_j summed left to right, then y0 + sum), in fp32
            if (NK > 0) {
#pragma unroll
                for (int q = 0; q < BQ; ++q) {
                    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int j = 0; j < NK; ++j) {
                        const float c = cf[j];
                        const float tx = __fmul_rn(c, kv[j][q].x), ty = __fmul_rn(c, kv[j][q].y);
                        const float tz = __fmul_rn(c, kv[j][q].z), tw = __fmul_rn(c, kv[j][q].w);
                        acc.x = j ? __fadd_rn(acc.x, tx) : tx;
                        acc.y = j ? __fadd_rn(acc.y, ty) : ty;
                        acc.z = j ? __fadd_rn(acc.z, tz) : tz;
                        acc.w = j ? __fadd_rn(acc.w, tw) : tw;
                    }
                    v[q].x = __fadd_rn(v[q].x, acc.x);
                    v[q].y = __fadd_rn(v[q].y, acc.y);
                    v[q].z = __fadd_rn(v[q].z, acc.z);
                    v[q].w = __fadd_rn(v[q].w, acc.w);
                    if (p.ystage && n0 == 0 && mode == 0 && in[q]) *reinterpret_cast<float4 *>(p.ystage + off[q]) = v[q];
                }
            }
#pragma unroll
            for (int q = 0; q < BQ; ++q) {
                const int f = tid + (b0 + q) * NTHR;
                const int row = f / (kKChunk / 4), c4 = f % (kKChunk / 4);
                const uint4 t = (mode == 1) ? make_uint4(tf32_lo(v[q].x), tf32_lo(v[q].y), tf32_lo(v[q].z), tf32_lo(v[q].w))
                                            : make_uint4(to_tf32(v[q].x), to_tf32(v[q].y), to_tf32(v[q].z), to_tf32(v[q].w));
                *reinterpret_cast<uint4 *>(sA + (c4 >> 3) * (kTileM * 128) + sw128_offset(row, c4 & 7)) = t;
            }
        }
    } else {
        for (int f = tid; f < kTileM * (kKChunk / 4); f += NTHR) {
            const int row = f / (kKChunk / 4), c4 = f % (kKChunk / 4);
            const int gm = m0 + row, gk = kc + c4 * 4;
            float e[4] = {0.f, 0.f, 0.f, 0.f};
            if (gm < p.M) {
                for (int q = 0; q < 4 && gk + q < p.K; ++q) {
                    const size_t off = (size_t)gm * p.K + gk + q;
                    float a = p.x[off];
                    if (NK > 0) {
                        float acc = 0.f;
#pragma unroll
                        for (int j = 0; j < NK; ++j) {
                            const float t = __fmul_rn(cf[j], p.k[j][off]);
                            acc = j ? __fadd_rn(acc, t) : t;
                        }
                        a = __fadd_rn(a, acc);
                        if (p.ystage && n0 == 0 && mode == 0) p.ystage[off] = a;
                    }
                    e[q] = a;
                }
            }
            const uint4 t = (mode == 1) ? make_uint4(tf32_lo(e[0]), tf32_lo(e[1]), tf32_lo(e[2]), tf32_lo(e[3]))
                                        : make_uint4(to_tf32(e[0]), to_tf32(e[1]), to_tf32(e[2]), to_tf32(e[3]));
            *reinterpret_cast<uint4 *>(sA + (c4 >> 3) * (kTileM * 128) + sw128_offset(row, c4 & 7)) = t;
        }
    }
}

template <int NTHR>
__device__ __forceinline__ void produce_chunk(const DenseParams &p, uint8_t *sA, uint8_t *sB, int m0, int n0, int NT, int kc,
                                              int tid, const float (&cf)[kMaxNK], int mode = 0) {
    switch (p.nk) {
        case 0: produce_chunk_t<NTHR, 0>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
        case 1: produce_chunk_t<NTHR, 1>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
        case 2: produce_chunk_t<NTHR, 2>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
        case 3: produce_chunk_t<NTHR, 3>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
        case 4: produce_chunk_t<NTHR, 4>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
        case 5: produce_chunk_t<NTHR, 5>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
        case 6: produce_chunk_t<NTHR, 6>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
        case 7: produce_chunk_t<NTHR, 7>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
        default: produce_chunk_t<NTHR, 8>(p, sA, sB, m0, n0, NT, kc, tid, cf, mode); break;
    }
}

// ================================================================================================
// k_dense_layer_tf32: persistent, one CTA per SM, items = (128-row tile, 64 NS-column tile).  A two-stage ring of
// (A chunk, B chunk) shared-memory buffers: while the wgmmas of chunk c run asynchronously, all 256 threads produce chunk
// c + 1 into the other stage, then wait for the MMAs and hand the stage over with one CTA barrier.
// NS (1..4) is the number of 64-column MMAs per K step, i.e. the N tile is 64 NS wide (the last tile may be narrower:
// the columns past N read whatever the B stage holds and are never stored).
// ================================================================================================
constexpr int kStageBytesA = kTileM * 128 * 2;                    // 128 rows x 64 K columns = 32 KB
constexpr int kStageBytes = kStageBytesA + 256 * 128 * 2;         // + up to 256 rows of W x 64 K columns = 96 KB

template <int ACT, int NS>
__device__ __forceinline__ void dense_epilogue(const DenseParams &p, float (&acc)[4][32], int row_base, int n0, int NT, int lane) {
#pragma unroll
    for (int j = 0; j < NS; ++j)
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int col = j * kNSub + q * 8 + 2 * (lane & 3);
            if (col >= NT) continue;                                // NT is a multiple of 16: both columns of the pair
            const float b0 = p.bias ? p.bias[n0 + col] : 0.f, b1 = p.bias ? p.bias[n0 + col + 1] : 0.f;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int row = row_base + (lane >> 2) + 8 * i;
                if (row < p.M)
                    *reinterpret_cast<float2 *>(p.out + (size_t)row * p.N + n0 + col) =
                        make_float2(act_t<ACT>(acc[j][q * 4 + 2 * i] + b0), act_t<ACT>(acc[j][q * 4 + 2 * i + 1] + b1));
            }
        }
}

template <int NS>
__global__ void __launch_bounds__(kConsumerThreads, 1) k_dense_layer_tf32(const __grid_constant__ DenseParams p) {
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the swizzle atoms
    uint8_t *smem = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31, wq = (tid >> 5) & 3;
    constexpr int NTILE = NS * kNSub;
    const int tiles_m = (p.M + kTileM - 1) / kTileM;
    const int tiles_n = (p.N + NTILE - 1) / NTILE;
    const int items = tiles_m * tiles_n;
    const int kchunks = (p.K + kKChunk - 1) / kKChunk;
    const int chunks = p.W_lo ? 3 * kchunks : kchunks;      // 3xTF32: three passes over K (A_lo.W_hi, A_hi.W_lo, A_hi.W_hi)

    float cf[kMaxNK];
#pragma unroll
    for (int j = 0; j < kMaxNK; ++j) cf[j] = 0.f;
    if (p.nk > 0) {
        const float dt = (float)p.st->dt;
#pragma unroll
        for (int j = 0; j < kMaxNK; ++j)
            if (j < p.nk) cf[j] = __fmul_rn(dt, (float)p.coef[j]);
    }
    const uint32_t smem_lo = desc_lo(smem_u32(smem));

    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int m0 = (item / tiles_n) * kTileM, n0 = (item % tiles_n) * NTILE;
        const int NT = (p.N - n0) < NTILE ? (p.N - n0) : NTILE;
        auto produce = [&](int c) {
            const int pass = c / kchunks;
            const int mode = p.W_lo ? (pass == 0 ? 1 : pass == 1 ? 2 : 0) : 0;
            uint8_t *sA = smem + (c & 1) * kStageBytes;
            produce_chunk<kConsumerThreads>(p, sA, sA + kStageBytesA, m0, n0, NT, (c - pass * kchunks) * kKChunk, tid, cf, mode);
        };
        produce(0);
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        // make the generic-proxy writes visible to the tensor core (async proxy), then hand over
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        float acc[4][32];
        for (int c = 0; c < chunks; ++c) {
            const uint32_t a_lo = smem_lo + (uint32_t)((c & 1) * kStageBytes + wg * 64 * 128) / 16u;
            const uint32_t b_lo = smem_lo + (uint32_t)((c & 1) * kStageBytes + kStageBytesA) / 16u;
            wgmma_fence();
            fence_acc<NS>(acc);
            mma_kblock<NS>(acc, a_lo, b_lo, c > 0);
            mma_kblock<NS>(acc, a_lo + (kTileM * 128) / 16, b_lo + (256 * 128) / 16, true);
            wgmma_commit();
            if (c + 1 < chunks) produce(c + 1);                     // overlaps the MMAs just issued
            wgmma_wait<0>();
            fence_acc<NS>(acc);
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
        }
        const int row_base = m0 + wg * 64 + wq * 16;
        switch (p.act) {
            case 1: dense_epilogue<1, NS>(p, acc, row_base, n0, NT, lane); break;
            case 2: dense_epilogue<2, NS>(p, acc, row_base, n0, NT, lane); break;
            case 3: dense_epilogue<3, NS>(p, acc, row_base, n0, NT, lane); break;
            default: dense_epilogue<0, NS>(p, acc, row_base, n0, NT, lane); break;
        }
    }
}

// ================================================================================================
// The whole ODENet-style func in ONE kernel: fc1 -> act -> fc2 -> act -> fc3 chained per 128-row tile, the hidden
// activations never leave the SM.
//
//   ACT   : 128 rows x up to 256 TF32 columns of shared memory (<= 128 KB), the A operand of whichever GEMM is running:
//           first the (optionally stage-combined) input tile, then act(h1), then act(h2) -- each written in the K-major
//           SWIZZLE_128B layout.  Warpgroup g's GEMMs read only its own 64 rows, so after the first GEMM each warpgroup
//           overwrites its rows with the next activation as soon as its own MMAs are done (no CTA-wide barrier)
//   ring  : S stages x [N rows x 32 columns] of the current layer's weights.  The weights are packed ONCE per weight
//           version (k_mlp3_pack) into exactly this shared-memory image -- TF32-rounded, swizzled, zero-padded -- so one
//           thread streams them with cp.async.bulk (the TMA engine's linear mode) and an mbarrier transaction count
//   warps : 0-7 two consumer warpgroups (input tile, wgmma with register accumulators, bias / activation epilogues),
//           8 weight loader.  A stage goes back to the loader when both warpgroups' MMAs on it have completed.
// HBM traffic per evaluation: the input tile(s) and the output tile -- (1 + nk) x 4D + 4D bytes per row instead of
// 4(D + 4H + D) bytes per row through three separate layers; the weights stream from L2.
// ================================================================================================
constexpr int kSub = 32;                                   // K columns per weight sub-chunk (one 128-byte swizzle row)
// + the weight-loader warp.  9 warps put 3 on one quarter of the SM's register file: at most 168 registers per thread
// for 128 accumulators and everything else (ptxas spills a few values, reloaded outside the MMA loop)
constexpr int kMlp3Threads = kConsumerThreads + 32;
constexpr int kMaxRing = 8;
constexpr uint32_t kBulkPiece = 16384;                     // bytes per cp.async.bulk request
// a 64-column MMA over a layer narrower than 64 NS reads up to 48 rows (6 KB) past the stage; keep that inside the allocation
constexpr int kRingTail = 8192;

struct Mlp3Params {
    DenseParams in;                    // x / k / coef / nk / st / ystage / M / K(= D) describe the input tile
    const uint8_t *packed;             // k_mlp3_pack's image: layer 1 sub-chunks, layer 2, layer 3
    const float *b1, *b2, *b3;
    float *out;                        // [M, D]
    int M, D, H, act;
    int act_bytes, stage_bytes, stages;
};

__host__ __device__ inline int mlp3_subs(int K) { return (K + kSub - 1) / kSub; }
__host__ __device__ inline size_t mlp3_layer_bytes(int N, int K) { return (size_t)mlp3_subs(K) * N * 128; }

// TF32-round, swizzle and zero-pad W[N, K] into sub-chunk images of [N rows x 128 B]
__global__ void k_mlp3_pack(const float *W1, const float *W2, const float *W3, int D, int H, uint8_t *packed) {
    const size_t n1 = mlp3_layer_bytes(H, D) / 16, n2 = mlp3_layer_bytes(H, H) / 16, n3 = mlp3_layer_bytes(D, H) / 16;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2 + n3; i += (size_t)gridDim.x * blockDim.x) {
        const float *W;
        int N, K;
        size_t j = i;
        if (j < n1) {
            W = W1, N = H, K = D;
        } else if (j < n1 + n2) {
            W = W2, N = H, K = H, j -= n1;
        } else {
            W = W3, N = D, K = H, j -= n1 + n2;
        }
        const int q = (int)(j & 7);                       // 16-byte slot inside the 128-byte row of the image
        const int row = (int)((j >> 3) % N);
        const int c = (int)((j >> 3) / N);
        const int piece = q ^ (row & 7);                  // which 4 source columns live in that slot (Swizzle<3,4,3>)
        uint32_t e[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int gk = c * kSub + piece * 4 + u;
            e[u] = gk < K ? to_tf32(W[(size_t)row * K + gk]) : 0u;
        }
        reinterpret_cast<uint4 *>(packed)[i] = make_uint4(e[0], e[1], e[2], e[3]);
    }
}

// One layer's GEMM for this warpgroup: acc (64 rows x Nl columns) = ACT[rows of the warpgroup, 0:32 nsub] . W^T, the weight
// K blocks taken from the ring in stage order.  The wgmmas of a stage run while the next stage is awaited; a stage is
// released (one arrival per warpgroup on its `empty` barrier) once the MMAs that read it have completed.
template <int NS>
__device__ __forceinline__ void mlp3_gemm(float (&acc)[4][32], uint32_t a_lo, uint32_t ring_lo, int Nl, int nsub, int stage_bytes,
                                          uint32_t S, uint32_t &it, uint64_t *bar_full, uint64_t *bar_empty, bool leader) {
    const int grp = stage_bytes / (Nl * 128);                    // K blocks per stage (narrow layers: several)
    uint32_t prev = 0xffffffffu;
    for (int c = 0; c < nsub; c += grp, ++it) {
        const uint32_t s = it % S, ph = (it / S) & 1u;
        const int nb = nsub - c < grp ? nsub - c : grp;
        mbar_wait(smem_u32(&bar_full[s]), ph);
        wgmma_fence();
        fence_acc<NS>(acc);
        const uint32_t b_lo = ring_lo + s * ((uint32_t)stage_bytes >> 4);
        for (int kb = 0; kb < nb; ++kb)
            mma_kblock<NS>(acc, a_lo + (uint32_t)(c + kb) * ((kTileM * 128) >> 4), b_lo + (uint32_t)kb * ((uint32_t)(Nl * 128) >> 4),
                           (c + kb) > 0);
        wgmma_commit();
        wgmma_wait<1>();                                           // the previous stage's MMAs are done
        if (leader && prev != 0xffffffffu) mbar_arrive(smem_u32(&bar_empty[prev]));
        prev = s;
    }
    wgmma_wait<0>();
    fence_acc<NS>(acc);
    if (leader) mbar_arrive(smem_u32(&bar_empty[prev]));
}

__device__ __forceinline__ void mlp3_gemm_n(float (&acc)[4][32], int ns, uint32_t a_lo, uint32_t ring_lo, int Nl, int nsub,
                                            int stage_bytes, uint32_t S, uint32_t &it, uint64_t *bar_full, uint64_t *bar_empty,
                                            bool leader) {
    switch (ns) {
        case 1: mlp3_gemm<1>(acc, a_lo, ring_lo, Nl, nsub, stage_bytes, S, it, bar_full, bar_empty, leader); break;
        case 2: mlp3_gemm<2>(acc, a_lo, ring_lo, Nl, nsub, stage_bytes, S, it, bar_full, bar_empty, leader); break;
        case 3: mlp3_gemm<3>(acc, a_lo, ring_lo, Nl, nsub, stage_bytes, S, it, bar_full, bar_empty, leader); break;
        default: mlp3_gemm<4>(acc, a_lo, ring_lo, Nl, nsub, stage_bytes, S, it, bar_full, bar_empty, leader); break;
    }
}

// bias + activation + TF32 rounding of this warpgroup's accumulator fragment, written into its rows of ACT as the next
// GEMM's A operand; columns from ncols up to the next multiple of 32 are written as zeros (the K padding).
// Fragment element (row_base + l / 4 + 8i, 64j + 8q + 2 (l % 4) + c) lands in K block 2j + q / 4, row atom row_base / 8 + i,
// atom row l / 4, 16-byte chunk (2 (q % 4) + (l % 4) / 2) XOR (l / 4), word 2 (l % 2) + c: one per-thread base and a XOR
// term, the rest compile-time constants (computing sw128_offset per element made ptxas keep 64 addresses live and spill).
template <int ACT, int NS>
__device__ __forceinline__ void epilogue_to_act_t(uint8_t *act_buf, const float (&acc)[4][32], int row_base, int lane, int ncols,
                                                  const float *bias) {
    const int ncols_pad = (ncols + kSub - 1) / kSub * kSub;
    const int rx = lane >> 2;
    const uint32_t t = (uint32_t)(((lane & 3) >> 1) ^ rx);
    uint8_t *base = act_buf + (row_base >> 3) * 1024 + rx * 128 + (lane & 1) * 8;
#pragma unroll
    for (int j = 0; j < NS; ++j)
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int col = j * kNSub + q * 8 + 2 * (lane & 3);
            if (j * kNSub + q * 8 >= ncols_pad) continue;              // warp-uniform: ncols_pad is a multiple of 32
            const bool in = col < ncols;                              // ncols is a multiple of 16: both columns of the pair
            const float b0 = bias[col], b1 = bias[col + 1];
            uint8_t *blk = base + (2 * j + (q >> 2)) * (kTileM * 128) + ((((uint32_t)(2 * (q & 3))) ^ t) << 4);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const uint32_t v0 = in ? to_tf32_fast(act_t<ACT>(acc[j][q * 4 + 2 * i] + b0)) : 0u;
                const uint32_t v1 = in ? to_tf32_fast(act_t<ACT>(acc[j][q * 4 + 2 * i + 1] + b1)) : 0u;
                *reinterpret_cast<uint2 *>(blk + i * 1024) = make_uint2(v0, v1);
            }
        }
}

template <int NS>
__device__ __forceinline__ void epilogue_to_act_n(uint8_t *act_buf, const float (&acc)[4][32], int row_base, int lane, int ncols,
                                                  const float *bias, int act) {
    switch (act) {
        case 1: epilogue_to_act_t<1, NS>(act_buf, acc, row_base, lane, ncols, bias); break;
        case 2: epilogue_to_act_t<2, NS>(act_buf, acc, row_base, lane, ncols, bias); break;
        case 3: epilogue_to_act_t<3, NS>(act_buf, acc, row_base, lane, ncols, bias); break;
        default: epilogue_to_act_t<0, NS>(act_buf, acc, row_base, lane, ncols, bias); break;
    }
}

__device__ __forceinline__ void epilogue_to_act(uint8_t *act_buf, const float (&acc)[4][32], int ns, int row_base, int lane, int ncols,
                                                const float *bias, int act) {
    switch (ns) {
        case 1: epilogue_to_act_n<1>(act_buf, acc, row_base, lane, ncols, bias, act); break;
        case 2: epilogue_to_act_n<2>(act_buf, acc, row_base, lane, ncols, bias, act); break;
        case 3: epilogue_to_act_n<3>(act_buf, acc, row_base, lane, ncols, bias, act); break;
        default: epilogue_to_act_n<4>(act_buf, acc, row_base, lane, ncols, bias, act); break;
    }
}

// output tile: accumulator (D columns) + bias -> global rows of this warpgroup
template <int NS>
__device__ __forceinline__ void output_tile_t(const Mlp3Params &P, const float (&acc)[4][32], int row_base, int lane, const float *bias) {
#pragma unroll
    for (int j = 0; j < NS; ++j)
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int col = j * kNSub + q * 8 + 2 * (lane & 3);
            if (col >= P.D) continue;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int row = row_base + (lane >> 2) + 8 * i;
                if (row < P.M)
                    *reinterpret_cast<float2 *>(P.out + (size_t)row * P.D + col) =
                        make_float2(acc[j][q * 4 + 2 * i] + bias[col], acc[j][q * 4 + 2 * i + 1] + bias[col + 1]);
            }
        }
}

__device__ __forceinline__ void output_tile(const Mlp3Params &P, const float (&acc)[4][32], int ns, int row_base, int lane,
                                            const float *bias) {
    switch (ns) {
        case 1: output_tile_t<1>(P, acc, row_base, lane, bias); break;
        case 2: output_tile_t<2>(P, acc, row_base, lane, bias); break;
        case 3: output_tile_t<3>(P, acc, row_base, lane, bias); break;
        default: output_tile_t<4>(P, acc, row_base, lane, bias); break;
    }
}

__global__ void __launch_bounds__(kMlp3Threads, 1) k_mlp3_tf32(const __grid_constant__ Mlp3Params P) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t *act_buf = smem;
    uint8_t *ring = smem + P.act_bytes;
    __shared__ __align__(8) uint64_t bar_full[kMaxRing], bar_empty[kMaxRing];
    __shared__ __align__(16) float sbias[3][256];

    const DenseParams &p = P.in;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int D = P.D, H = P.H;
    for (int i = tid; i < 3 * 256; i += kMlp3Threads) {
        const int l = i >> 8, c = i & 255;
        const float *b = l == 0 ? P.b1 : (l == 1 ? P.b2 : P.b3);
        sbias[l][c] = (b && c < (l == 2 ? D : H)) ? b[c] : 0.f;
    }
    const int tiles_m = (P.M + kTileM - 1) / kTileM;
    const int sub1 = mlp3_subs(D), sub2 = mlp3_subs(H);
    const uint32_t S = (uint32_t)P.stages;
    if (tid == 0) {
        for (int i = 0; i < kMaxRing; ++i) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&bar_full[i])), "r"(1u));   // loader's expect_tx arrive + the bytes
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&bar_empty[i])), "r"(2u));  // one arrival per consumer warpgroup
        }
        asm volatile("fence.mbarrier_init.release.cluster;");
    }
    __syncthreads();

    if (warp == kConsumerThreads / 32) {
        // ===== weight loader: one bulk copy per piece, completion counted in bytes on the stage's mbarrier =====
        if (lane == 0) {
            uint32_t it = 0;
            for (int tile = blockIdx.x; tile < tiles_m; tile += gridDim.x) {
                const uint8_t *src = P.packed;
                for (int l = 0; l < 3; ++l) {
                    const int Nl = l == 2 ? D : H;
                    const int nsub = l == 0 ? sub1 : sub2;
                    const int grp = P.stage_bytes / (Nl * 128);
                    for (int c = 0; c < nsub; c += grp, ++it) {
                        const uint32_t bytes = (uint32_t)((nsub - c < grp ? nsub - c : grp) * Nl) * 128u;
                        const uint32_t s = it % S, ph = (it / S) & 1u;
                        mbar_wait(smem_u32(&bar_empty[s]), ph ^ 1u);
                        const uint32_t bar = smem_u32(&bar_full[s]);
                        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
                        const uint32_t dst0 = smem_u32(ring + (size_t)s * P.stage_bytes);
                        for (uint32_t o = 0; o < bytes; o += kBulkPiece) {
                            const uint32_t nb = bytes - o < kBulkPiece ? bytes - o : kBulkPiece;
                            asm volatile(
                                "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst0 + o),
                                "l"(src + o), "r"(nb), "r"(bar)
                                : "memory");
                        }
                        src += bytes;
                    }
                }
            }
        }
        return;
    }

    // ===== consumer warpgroups =====
    const int wg = tid >> 7, wq = (tid >> 5) & 3;
    const bool leader = (tid & (kWgThreads - 1)) == 0;
    const int nsH = (H + kNSub - 1) / kNSub, nsD = (D + kNSub - 1) / kNSub;
    const uint32_t act_lo = desc_lo(smem_u32(act_buf)) + (uint32_t)(wg * 64 * 128) / 16u;   // this warpgroup's 64 rows
    const uint32_t ring_lo = desc_lo(smem_u32(ring));
    const int row_in_tile = wg * 64 + wq * 16;
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < tiles_m; tile += gridDim.x) {
        const int m0 = tile * kTileM;
        float cf[kMaxNK];                                        // (per tile: not held across the GEMMs)
#pragma unroll
        for (int j = 0; j < kMaxNK; ++j) cf[j] = 0.f;
        if (p.nk > 0) {
            const float dt = (float)p.st->dt;
#pragma unroll
            for (int j = 0; j < kMaxNK; ++j)
                if (j < p.nk) cf[j] = __fmul_rn(dt, (float)p.coef[j]);
        }
        consumers_sync();                                        // both warpgroups' GEMM3 of the previous tile are done with ACT
        for (int kc = 0; kc < D; kc += kKChunk)
            produce_chunk<kConsumerThreads>(p, act_buf + (kc / kSub) * (kTileM * 128), nullptr, m0, 0, 0, kc, tid, cf);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        consumers_sync();
        float acc[4][32];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int r = 0; r < 32; ++r) acc[j][r] = 0.f;          // (ends the registers' live range across the input load)
        // h1 = act(x W1^T + b1) -> ACT
        mlp3_gemm_n(acc, nsH, act_lo, ring_lo, H, sub1, P.stage_bytes, S, it, bar_full, bar_empty, leader);
        epilogue_to_act(act_buf, acc, nsH, row_in_tile, lane, H, sbias[0], P.act);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        warpgroup_sync(wg);
        // h2 = act(h1 W2^T + b2) -> ACT
        mlp3_gemm_n(acc, nsH, act_lo, ring_lo, H, sub2, P.stage_bytes, S, it, bar_full, bar_empty, leader);
        epilogue_to_act(act_buf, acc, nsH, row_in_tile, lane, H, sbias[1], P.act);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        warpgroup_sync(wg);
        // out = h2 W3^T + b3
        mlp3_gemm_n(acc, nsD, act_lo, ring_lo, D, sub2, P.stage_bytes, S, it, bar_full, bar_empty, leader);
        output_tile(P, acc, nsD, m0 + row_in_tile, lane, sbias[2]);
    }
}

// ================================================================================================
// k_linear_f64: the linear right-hand side  out[M, D] = Y[M, D] . A[D, D]  on the fp64 tensor cores, where Y = x or
// the Runge-Kutta stage input formed on the fly, Y = x + sum_j (dt * coef_j) k_j.  wgmma has no fp64 form; the fp64
// tensor path of sm_90 is mma.sync m16n8k16 (DMMA), fp64 accumulators in registers.
//
//   persistent: one CTA of 8 warps per SM.  A's image (<= 128 KB) is copied into shared memory once per CTA; a warp
//               then walks 16-row blocks of Y (block b, b + 8 gridDim, ...) and computes all D output columns of each
//   operands  : the A fragment comes straight from global memory into registers -- a thread loads 4 consecutive
//               doubles of its two rows per 16-column K chunk (two 16-byte loads per row, a warp's loads cover 16
//               whole 128-byte row segments), forms the stage combine there and feeds the DMMAs; Y never goes
//               through shared memory and never reaches HBM unless `ystage` asks for it.  K inside a chunk is
//               permuted (PTX's k = tig + 4u is column 4 tig + u of the chunk); the image holds the rows of A in the
//               same permutation, so the product is unchanged
//   image     : [D/16 chunks][D/8 n tiles][2 halves][32 lanes][2] doubles, lane l = 4 g + tig of the half h holding
//               A[16 c + 4 tig + 2 h + e][8 n + g]: a B fragment is two 16-byte shared loads over 512 contiguous bytes
//               per warp -- no bank conflicts.  A pure permutation (and sign) of A, built by rhs.py with torch ops
//   pipeline  : NK <= 1: the raw loads of the next K chunk (of this row block or of the next one) are issued before the
//               current chunk's DMMAs, so HBM latency hides behind the tensor core.  NK >= 2: the (1 + NK) streams of a
//               chunk are already several KB in flight per warp; they are loaded in batches of kLinBatch k's, combined
//               in order as each batch arrives
//   order     : every row block runs the same instruction sequence: chunks in increasing K, one DMMA per (chunk, n
//               tile), whatever M, nk, the row's position or the CTA.  A row's result depends only on that row's input
//               (and A), so fused and unfused evaluations, and any split of the rows over launches or GPUs, agree bit
//               for bit.  The combine is k_rk_stage's: c_j = dt * coef_j, acc = c_0 k_0, acc += c_j k_j left to right,
//               Y = x + acc, round-to-nearest multiplies and adds with no contraction.
// ================================================================================================
constexpr int kLinWarps = 8;
constexpr int kLinThreads = kLinWarps * 32;
constexpr int kLinMaxD = 128;
constexpr int kLinMaxNK = B2ODE_MAXK - 1;      // a stage row of a 14-stage tableau has at most 13 terms
constexpr int kLinBatch = 2;                   // k streams loaded per batch when NK >= 2

struct LinearParams {
    const double *x;                     // [M, D]: Y (nk == 0) or y0 of the step
    const double *k[kLinMaxNK];          // stage derivatives [M, D]
    double coef[kLinMaxNK];              // beta_j of the stage row (zeros already dropped)
    int nk;
    const b2ode_state *st;               // dt lives here when nk > 0
    double *ystage;                      // optional: also store Y
    const double *image;                 // A's shared-memory image (see above)
    double *out;                         // [M, D]
    int M, D;
};

// D[16 x 8] += A[16 x 16] . B[16 x 8], fp64.  Fragments (g = lane / 4, tig = lane % 4): a[2u + r] = A[g + 8r][tig + 4u],
// b[i] = B[tig + 4i][g], d[2r + c] = D[g + 8r][2 tig + c]
__device__ __forceinline__ void dmma_m16n8k16(double (&d)[4], const double (&a)[8], double b0, double b1, double b2, double b3) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
        "{%12, %13, %14, %15}, {%0, %1, %2, %3};"
        : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b0), "d"(b1), "d"(b2), "d"(b3));
}

// 4 consecutive doubles of one row (two 16-byte loads), zeros for a row past M
__device__ __forceinline__ void lin_load4(double (&v)[4], const double *src, bool in) {
    double2 lo = make_double2(0.0, 0.0), hi = make_double2(0.0, 0.0);
    if (in) {
        lo = *reinterpret_cast<const double2 *>(src);
        hi = *reinterpret_cast<const double2 *>(src + 2);
    }
    v[0] = lo.x, v[1] = lo.y, v[2] = hi.x, v[3] = hi.y;
}

template <int NK>
__global__ void __launch_bounds__(kLinThreads, 1) k_linear_f64(const __grid_constant__ LinearParams p) {
    extern __shared__ __align__(16) double s_img[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, tig = lane & 3;
    const int D = p.D, KC = D >> 4, NT = D >> 3;
    {
        const double2 *src = reinterpret_cast<const double2 *>(p.image);
        double2 *dst = reinterpret_cast<double2 *>(s_img);
        for (int i = tid; i < (D * D) >> 1; i += kLinThreads) dst[i] = src[i];
    }
    double c[NK > 0 ? NK : 1];
    if (NK > 0) {
        const double dt = p.st->dt;
#pragma unroll
        for (int j = 0; j < NK; ++j) c[j] = Ar<double>::mul(dt, p.coef[j]);
    }
    __syncthreads();

    const long long blocks = ((long long)p.M + 15) >> 4;
    const long long stride = (long long)gridDim.x * kLinWarps;
    // element offset of this thread's 4 columns of K chunk kc in row block b: row 16 b + g (+ 8 * r), column 16 kc + 4 tig
    auto offset = [&](long long b, int kc, int r) { return (b * 16 + g + 8 * r) * (long long)D + kc * 16 + tig * 4; };
    auto row_in = [&](long long b, int r) { return b * 16 + g + 8 * r < p.M; };

    constexpr bool kPrefetch = NK <= 1;
    double nx[2][NK + 1][4];                 // prefetched raw chunk: [row r][stream: x, k_0][4 columns]
    long long b = (long long)blockIdx.x * kLinWarps + warp;
    if (kPrefetch && b < blocks) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const long long o = offset(b, 0, r);
            lin_load4(nx[r][0], p.x + o, row_in(b, r));
#pragma unroll
            for (int j = 0; j < NK; ++j) lin_load4(nx[r][j + 1], p.k[j] + o, row_in(b, r));
        }
    }
    for (; b < blocks; b += stride) {
        double acc[kLinMaxD / 8][4];
#pragma unroll
        for (int n = 0; n < kLinMaxD / 8; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.0;
        const bool in0 = row_in(b, 0), in1 = row_in(b, 1);
#pragma unroll 1
        for (int kc = 0; kc < KC; ++kc) {
            double y[2][4];
            if (kPrefetch) {
                double cur[2][NK + 1][4];
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int s = 0; s <= NK; ++s)
#pragma unroll
                        for (int e = 0; e < 4; ++e) cur[r][s][e] = nx[r][s][e];
                // next chunk: this row block's, or the first chunk of the warp's next row block
                const long long nb = kc + 1 < KC ? b : b + stride;
                const int nkc = kc + 1 < KC ? kc + 1 : 0;
                if (nb < blocks) {
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const long long o = offset(nb, nkc, r);
                        lin_load4(nx[r][0], p.x + o, row_in(nb, r));
#pragma unroll
                        for (int j = 0; j < NK; ++j) lin_load4(nx[r][j + 1], p.k[j] + o, row_in(nb, r));
                    }
                }
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        y[r][e] = NK == 0 ? cur[r][0][e] : Ar<double>::add(cur[r][0][e], Ar<double>::mul(c[0], cur[r][NK > 0 ? 1 : 0][e]));
            } else {
                // y0 with the first batch of k's, then further batches; the sum runs left to right across batches
                double acc_c[2][4];
#pragma unroll
                for (int j0 = 0; j0 < NK; j0 += kLinBatch) {
                    constexpr int kB = kLinBatch;
                    double kv[kB][2][4];
                    const int nb = NK - j0 < kB ? NK - j0 : kB;
                    if (j0 == 0) {
#pragma unroll
                        for (int r = 0; r < 2; ++r) lin_load4(y[r], p.x + offset(b, kc, r), r ? in1 : in0);
                    }
#pragma unroll
                    for (int q = 0; q < kB; ++q)
                        if (q < nb)
#pragma unroll
                            for (int r = 0; r < 2; ++r) lin_load4(kv[q][r], p.k[j0 + q] + offset(b, kc, r), r ? in1 : in0);
#pragma unroll
                    for (int q = 0; q < kB; ++q)
                        if (q < nb)
#pragma unroll
                            for (int r = 0; r < 2; ++r)
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const double t = Ar<double>::mul(c[j0 + q], kv[q][r][e]);
                                    acc_c[r][e] = (j0 + q) ? Ar<double>::add(acc_c[r][e], t) : t;
                                }
                }
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int e = 0; e < 4; ++e) y[r][e] = Ar<double>::add(y[r][e], acc_c[r][e]);
            }
            if (NK > 0 && p.ystage) {
#pragma unroll
                for (int r = 0; r < 2; ++r)
                    if (r ? in1 : in0) {
                        double *dst = p.ystage + offset(b, kc, r);
                        *reinterpret_cast<double2 *>(dst) = make_double2(y[r][0], y[r][1]);
                        *reinterpret_cast<double2 *>(dst + 2) = make_double2(y[r][2], y[r][3]);
                    }
            }
            const double a[8] = {y[0][0], y[1][0], y[0][1], y[1][1], y[0][2], y[1][2], y[0][3], y[1][3]};
            const double2 *bimg = reinterpret_cast<const double2 *>(s_img) + (size_t)kc * NT * 64 + lane;
#pragma unroll
            for (int n = 0; n < kLinMaxD / 8; ++n)
                if (n < NT) {
                    const double2 b01 = bimg[n * 64], b23 = bimg[n * 64 + 32];
                    dmma_m16n8k16(acc[n], a, b01.x, b01.y, b23.x, b23.y);
                }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (!(r ? in1 : in0)) continue;
            double *dst = p.out + (b * 16 + g + 8 * r) * (long long)D + 2 * tig;
#pragma unroll
            for (int n = 0; n < kLinMaxD / 8; ++n)
                if (n < NT) *reinterpret_cast<double2 *>(dst + n * 8) = make_double2(acc[n][2 * r], acc[n][2 * r + 1]);
        }
    }
}

// ================================================================================================
// host side
// ================================================================================================
// cudaFuncSetAttribute is per device and the persistent grids are sized from the SM count: keep both per device ordinal
// (a process may drive several GPUs)
constexpr int kMaxDev = 64;
struct MmaDevCfg {
    bool dense[5], mlp3, linear[kLinMaxNK + 1];
    int sms;
};
static MmaDevCfg g_mma_dev[kMaxDev];

static int mma_dev(MmaDevCfg **cfg) {
    int dev = 0;
    B2_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= kMaxDev) return b2_fail(B2ODE_EINVAL, "device ordinal %d out of range", dev);
    MmaDevCfg *c = &g_mma_dev[dev];
    if (c->sms == 0) B2_CUDA(cudaDeviceGetAttribute(&c->sms, cudaDevAttrMultiProcessorCount, dev));
    *cfg = c;
    return 0;
}

static bool aligned16p(const void *p) { return ((uintptr_t)p & 15) == 0; }

// the producers' vector paths (see DenseParams::vec_a / vec_w); the scalar paths give the same bits
static void set_vector_paths(DenseParams &p) {
    bool a = (p.K & 3) == 0 && aligned16p(p.x) && aligned16p(p.ystage);
    for (int j = 0; j < p.nk; ++j) a = a && aligned16p(p.k[j]);
    p.vec_a = a;
    p.vec_w = (p.K & 3) == 0 && aligned16p(p.W) && aligned16p(p.W_lo);
}

template <int NS>
static int launch_dense(const DenseParams &p, MmaDevCfg *dc, cudaStream_t st) {
    const size_t smem = 2 * (size_t)kStageBytes + 1024;          // 2 x 96 KB ring + alignment slack
    if (!dc->dense[NS]) {
        B2_CUDA(cudaFuncSetAttribute(k_dense_layer_tf32<NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        dc->dense[NS] = true;
    }
    const long long items = ((p.M + kTileM - 1) / kTileM) * (long long)((p.N + NS * kNSub - 1) / (NS * kNSub));
    const int grid = (int)(items < dc->sms ? items : dc->sms);         // persistent: one CTA per SM
    k_dense_layer_tf32<NS><<<grid, kConsumerThreads, smem, st>>>(p);
    return 0;
}

static int dense_layer_impl(const void *x, const void *const *k, const double *coef, int nk, const void *state,
                            void *ystage, const void *W, const void *W_lo, const void *bias, void *out, int64_t M, int K, int N,
                            int act, void *cuda_stream) {
    if (!x || !W || !out || M < 1 || K < 1 || N < 1) return b2_fail(B2ODE_EINVAL, "bad dense-layer arguments");
    if (N % 16 != 0) return b2_fail(B2ODE_EINVAL, "dense layer: N must be a multiple of 16 (got %d)", N);
    if (nk < 0 || nk > kMaxNK || (nk > 0 && (!k || !coef || !state))) return b2_fail(B2ODE_EINVAL, "bad stage-combine arguments");
    if (act < 0 || act > 3) return b2_fail(B2ODE_EINVAL, "unknown activation %d", act);
    if (M > (int64_t)2147483647 - kTileM) return b2_fail(B2ODE_EINVAL, "M too large");
    if ((uintptr_t)out & 7) return b2_fail(B2ODE_EINVAL, "dense layer: out must be 8-byte aligned (the epilogue stores column pairs)");
    DenseParams p;
    memset(&p, 0, sizeof(p));
    p.x = (const float *)x;
    for (int j = 0; j < nk; ++j) {
        if (!k[j]) return b2_fail(B2ODE_EINVAL, "k[%d] is null", j);
        p.k[j] = (const float *)k[j];
        p.coef[j] = coef[j];
    }
    p.nk = nk;
    p.st = (const b2ode_state *)state;
    p.ystage = (float *)ystage;
    p.W = (const float *)W;
    p.W_lo = (const float *)W_lo;
    p.bias = (const float *)bias;
    p.out = (float *)out;
    p.M = (int)M;
    p.K = K;
    p.N = N;
    p.act = act;
    set_vector_paths(p);
    MmaDevCfg *dc = nullptr;
    {
        const int rc = mma_dev(&dc);
        if (rc) return rc;
    }
    // N tile = the layer's width rounded up to 64 columns, at most 256 (wider layers take several N tiles)
    const int ns = N >= 256 ? 4 : (N + kNSub - 1) / kNSub;
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    int rc = 0;
    switch (ns) {
        case 1: rc = launch_dense<1>(p, dc, st); break;
        case 2: rc = launch_dense<2>(p, dc, st); break;
        case 3: rc = launch_dense<3>(p, dc, st); break;
        default: rc = launch_dense<4>(p, dc, st); break;
    }
    if (rc) return rc;
    B2_CUDA(cudaGetLastError());
    b2_count_launch();
    return 0;
}

extern "C" int b2ode_dense_layer(const void *x, const void *const *k, const double *coef, int nk, const void *state,
                                 void *ystage, const void *W, const void *bias, void *out, int64_t M, int K, int N, int act,
                                 void *cuda_stream) {
    return dense_layer_impl(x, k, coef, nk, state, ystage, W, nullptr, bias, out, M, K, N, act, cuda_stream);
}

// 3xTF32: W_hi = tf32(W), W_lo = tf32(W - W_hi), both [N, K]; the kernel splits A the same way on the fly and accumulates
// A_lo.W_hi + A_hi.W_lo + A_hi.W_hi in fp32 -- products as accurate as fp32 FMAs at three times the tensor-core work.
extern "C" int b2ode_dense_layer_x3(const void *x, const void *const *k, const double *coef, int nk, const void *state,
                                    void *ystage, const void *W_hi, const void *W_lo, const void *bias, void *out, int64_t M, int K,
                                    int N, int act, void *cuda_stream) {
    if (!W_lo) return b2_fail(B2ODE_EINVAL, "W_lo is null");
    return dense_layer_impl(x, k, coef, nk, state, ystage, W_hi, W_lo, bias, out, M, K, N, act, cuda_stream);
}

// ---- fc1 -> act -> fc2 -> act -> fc3 in one launch (tfdiffeq/models/dense_odenet.py:85-92); see k_mlp3_tf32 ----
static bool mlp3_dims_ok(int D, int H) { return D >= 16 && H >= 16 && D <= 256 && H <= 256 && D % 16 == 0 && H % 16 == 0; }

extern "C" int64_t b2ode_mlp3_packed_bytes(int D, int H) {
    if (!mlp3_dims_ok(D, H)) return -1;
    return (int64_t)(mlp3_layer_bytes(H, D) + mlp3_layer_bytes(H, H) + mlp3_layer_bytes(D, H));
}

extern "C" int b2ode_mlp3_pack(const void *W1, const void *W2, const void *W3, int D, int H, void *packed, void *cuda_stream) {
    if (!W1 || !W2 || !W3 || !packed) return b2_fail(B2ODE_EINVAL, "null pointer");
    if (!mlp3_dims_ok(D, H)) return b2_fail(B2ODE_EINVAL, "mlp3: dim and hidden must be multiples of 16 in [16, 256] (got %d, %d)", D, H);
    if ((uintptr_t)packed & 15) return b2_fail(B2ODE_EINVAL, "packed image must be 16-byte aligned");
    const int64_t pieces = b2ode_mlp3_packed_bytes(D, H) / 16;
    const int grid = (int)((pieces + 255) / 256);
    k_mlp3_pack<<<grid, 256, 0, (cudaStream_t)cuda_stream>>>((const float *)W1, (const float *)W2, (const float *)W3, D, H, (uint8_t *)packed);
    B2_CUDA(cudaGetLastError());
    b2_count_launch();
    return 0;
}

extern "C" int b2ode_mlp3(const void *x, const void *const *k, const double *coef, int nk, const void *state, void *ystage,
                          const void *packed, const void *b1, const void *b2, const void *b3, void *out, int64_t M, int D, int H,
                          int act, void *cuda_stream) {
    if (!x || !packed || !out || M < 1) return b2_fail(B2ODE_EINVAL, "bad mlp3 arguments");
    if (!mlp3_dims_ok(D, H)) return b2_fail(B2ODE_EINVAL, "mlp3: dim and hidden must be multiples of 16 in [16, 256] (got %d, %d)", D, H);
    if ((uintptr_t)packed & 15) return b2_fail(B2ODE_EINVAL, "packed image must be 16-byte aligned");
    if (nk < 0 || nk > kMaxNK || (nk > 0 && (!k || !coef || !state))) return b2_fail(B2ODE_EINVAL, "bad stage-combine arguments");
    if (act < 0 || act > 3) return b2_fail(B2ODE_EINVAL, "unknown activation %d", act);
    if (M > (int64_t)2147483647 - kTileM) return b2_fail(B2ODE_EINVAL, "M too large");
    if ((uintptr_t)out & 7) return b2_fail(B2ODE_EINVAL, "mlp3: out must be 8-byte aligned (the epilogue stores column pairs)");
    Mlp3Params P;
    memset(&P, 0, sizeof(P));
    P.in.x = (const float *)x;
    for (int j = 0; j < nk; ++j) {
        if (!k[j]) return b2_fail(B2ODE_EINVAL, "k[%d] is null", j);
        P.in.k[j] = (const float *)k[j];
        P.in.coef[j] = coef[j];
    }
    P.in.nk = nk;
    P.in.st = (const b2ode_state *)state;
    P.in.ystage = (float *)ystage;
    P.in.M = (int)M;
    P.in.K = D;
    P.in.N = H;
    set_vector_paths(P.in);                                       // (no W: the weights come from the packed image)
    P.packed = (const uint8_t *)packed;
    P.b1 = (const float *)b1;
    P.b2 = (const float *)b2;
    P.b3 = (const float *)b3;
    P.out = (float *)out;
    P.M = (int)M;
    P.D = D;
    P.H = H;
    P.act = act;
    // shared memory: ACT holds the whole activation tile (input chunks are produced 64 columns = 2 blocks at a time),
    // then the weight ring and the tail the narrow layers' 64-column MMAs may read past it
    const int blocks_in = 2 * ((D + kKChunk - 1) / kKChunk), blocks_h = mlp3_subs(H);
    const int slots = blocks_in > blocks_h ? blocks_in : blocks_h;
    P.act_bytes = slots * (kTileM * 128);
    P.stage_bytes = (H > D ? H : D) * 128;
    const int smem_max = 227 * 1024 - 4096;                       // static shared memory: biases and barriers
    const int budget = smem_max - 1024 - P.act_bytes - kRingTail;  // alignment slack
    int stages = budget / P.stage_bytes;
    if (stages > kMaxRing) stages = kMaxRing;
    if (stages < 2) return b2_fail(B2ODE_EINVAL, "mlp3: shared memory budget exhausted");
    P.stages = stages;
    const size_t smem = (size_t)P.act_bytes + (size_t)stages * P.stage_bytes + kRingTail + 1024;
    MmaDevCfg *dc = nullptr;
    {
        const int rc = mma_dev(&dc);
        if (rc) return rc;
    }
    if (!dc->mlp3) {
        B2_CUDA(cudaFuncSetAttribute(k_mlp3_tf32, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
        dc->mlp3 = true;
    }
    const long long tiles = (M + kTileM - 1) / kTileM;
    const int grid = (int)(tiles < dc->sms ? tiles : dc->sms);
    k_mlp3_tf32<<<grid, kMlp3Threads, smem, (cudaStream_t)cuda_stream>>>(P);
    B2_CUDA(cudaGetLastError());
    b2_count_launch();
    return 0;
}

// ---- linear right-hand side y @ A on the fp64 tensor cores; see k_linear_f64 ----
static bool linear_dim_ok(int D) { return D >= 16 && D <= kLinMaxD && D % 16 == 0; }

extern "C" int64_t b2ode_linear_image_bytes(int D) {
    if (!linear_dim_ok(D)) return -1;
    return (int64_t)D * D * (int64_t)sizeof(double);
}

template <int NK>
static int launch_linear(const LinearParams &p, MmaDevCfg *dc, cudaStream_t st) {
    const size_t smem = (size_t)p.D * p.D * sizeof(double);
    if (!dc->linear[NK]) {
        B2_CUDA(cudaFuncSetAttribute(k_linear_f64<NK>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(kLinMaxD * kLinMaxD * sizeof(double))));
        dc->linear[NK] = true;
    }
    const long long warps = ((long long)p.M + 15) / 16;
    const long long need = (warps + kLinWarps - 1) / kLinWarps;
    const int grid = (int)(need < dc->sms ? need : dc->sms);          // persistent: one CTA per SM
    k_linear_f64<NK><<<grid, kLinThreads, smem, st>>>(p);
    return 0;
}

extern "C" int b2ode_linear_f64(const void *x, const void *const *k, const double *coef, int nk, const void *state, void *ystage,
                                const void *A_image, void *out, int64_t M, int D, void *cuda_stream) {
    if (!x || !A_image || !out) return b2_fail(B2ODE_EINVAL, "linear: x, A_image and out must not be null");
    if (!linear_dim_ok(D)) return b2_fail(B2ODE_EINVAL, "linear: D must be a multiple of 16 in [16, %d] (got %d)", kLinMaxD, D);
    if (M < 1 || M > (int64_t)2147483647 - 16) return b2_fail(B2ODE_EINVAL, "linear: M out of range (%lld)", (long long)M);
    if (nk < 0 || nk > kLinMaxNK) return b2_fail(B2ODE_EINVAL, "linear: nk must be in [0, %d] (got %d)", kLinMaxNK, nk);
    if (nk > 0 && (!k || !coef || !state)) return b2_fail(B2ODE_EINVAL, "linear: a stage combine needs k, coef and state");
    if (!aligned16p(x) || !aligned16p(A_image) || !aligned16p(out) || !aligned16p(ystage) || !aligned16p(state))
        return b2_fail(B2ODE_EINVAL, "linear: x, A_image, out, ystage and state must be 16-byte aligned");
    LinearParams p;
    memset(&p, 0, sizeof(p));
    for (int j = 0; j < nk; ++j) {
        if (!k[j]) return b2_fail(B2ODE_EINVAL, "linear: k[%d] is null", j);
        if (!aligned16p(k[j])) return b2_fail(B2ODE_EINVAL, "linear: k[%d] must be 16-byte aligned", j);
        p.k[j] = (const double *)k[j];
        p.coef[j] = coef[j];
    }
    p.x = (const double *)x;
    p.nk = nk;
    p.st = (const b2ode_state *)state;
    p.ystage = (double *)ystage;
    p.image = (const double *)A_image;
    p.out = (double *)out;
    p.M = (int)M;
    p.D = D;
    MmaDevCfg *dc = nullptr;
    {
        const int rc = mma_dev(&dc);
        if (rc) return rc;
    }
    const cudaStream_t st = (cudaStream_t)cuda_stream;
    const int rc = dispatch_count(std::make_integer_sequence<int, kLinMaxNK + 1>{}, nk,
                                  [&](auto n) { return launch_linear<decltype(n)::value>(p, dc, st); },
                                  "linear: nk must be in [0, %d] (got %d)", kLinMaxNK, nk);
    if (rc) return rc;
    B2_CUDA(cudaGetLastError());
    b2_count_launch();
    return 0;
}
