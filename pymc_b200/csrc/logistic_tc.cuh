// Logistic GLM, tensor-core PERFORMANCE mode (BASELINE config 3): the two contractions of one batched leapfrog,
// eta = X beta  and  G = X^T (y - sigmoid(eta)),  on the Hopper tensor cores (wgmma.mma_async, operands staged in shared
// memory by TMA) instead of the fp64 DMMA path of dense.cuh.
//
// wgmma has no fp64 kind, so every fp64 operand is split into two fp16 pieces, v = hi + lo with hi = fp16(v) and
// lo = fp16(v - hi) (22 significant bits), and a product is evaluated as hi*hi + hi*lo + lo*hi in three f16 MMAs with fp32
// accumulation (the lo*lo term is below 2^-22 relative).  fp16 holds magnitudes 2^-14 .. 65504 only, so every operand is
// first scaled by an exact power of two: X column k by 2^sx[k] (once, at b200_model_set_precision), beta by 2^-sx[k] (which
// keeps eta) and then by 2^tau[c] per chain, each chosen so that the column / row maximum lies in [2^14, 2^15)
// (tc_split_exponent).  eta is unscaled by 2^-tau[c] in fp32 before the sigmoid, and the finish kernel
// (logistic_finish_fm_kernel) multiplies feature k's gradient by 2^-sx[k].  The accuracy is then independent of the data's
// scale: an entry keeps 22 bits down to 2^-14 of its row / column maximum, and an absolute floor of 2^-39 of it below that.
// fp32 accumulators only ever cover a bounded number of terms: X beta sums K = 128 terms, and the gradient accumulator is
// drained into fp64 registers every kTcDrain slabs, so fp32 rounding does not build up over the rows of X.  The small
// correction products (hi*lo, lo*hi) are issued first, while the accumulator is still small, and hi*hi last.
// Accuracy against the fp64 path is measured by tests/test_gpu_tc.py.  The fp64 DMMA kernel stays the parity mode.
//
// One CTA = 64 chains x a strided set of 128-row slabs of X; two consumer warpgroups and a producer warp.  Per slab:
//   TMA   : X_hi, X_lo slab [128 rows][128 features] fp16 -> smem (SWIZZLE_128B, two 64-column boxes each) + the slab's
//           128 labels (fp32), 2 stages
//   GEMM 1: warpgroup w: eta[c][i] = sum_k beta[c][k] X[i][k] for the slab rows 64w..64w+63 (m64n64k16; A = beta pieces,
//           B = X pieces, both K-major in smem); r = y - sigmoid(eta) and the log-likelihood terms from the accumulator
//           registers, in fp32; r split into fp16 pieces and stored as K-major tile [64 chains][128 rows] in smem
//   GEMM 2: warpgroup w: G[c][k] += sum_i r[c][i] X[i][k] for the features 64w..64w+63 (A = r pieces, B = the SAME X
//           bytes read MN-major: box w of the stage)
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace b200 {

constexpr int kTcRows = 128;      // rows of X per slab (N of GEMM 1 over both warpgroups, K of GEMM 2)
constexpr int kTcChains = 64;     // chains per CTA (M of both GEMMs)
constexpr int kTcK = 128;         // features (padded)
constexpr int kTcStages = 2;      // X slab stages in shared memory
constexpr int kTcConsumers = 256; // two warpgroups
constexpr int kTcThreads = 32 + kTcConsumers;  // producer warp + consumers
constexpr int kTcDrain = 2;       // slabs per fp32 gradient accumulation chunk
constexpr uint32_t kTcBlockBytes = kTcRows * 64 * 2;          // one [128 rows][64 cols] fp16 box = 16 KB
constexpr uint32_t kTcPieceBytes = 2 * kTcBlockBytes;         // one piece of a [128][128] slab = 32 KB
constexpr uint32_t kTcStageBytes = 2 * kTcPieceBytes;         // X_hi + X_lo = 64 KB
constexpr uint32_t kTcABlockBytes = kTcChains * 64 * 2;       // one [64 chains][64 k] fp16 box = 8 KB
constexpr uint32_t kTcAPieceBytes = 2 * kTcABlockBytes;       // one piece of a [64][128] operand tile = 16 KB
constexpr uint32_t kTcYBytes = kTcRows * sizeof(float);
constexpr size_t kTcSmemBytes = 1024 /*align*/ + 2 * kTcAPieceBytes /*beta*/ + 2 * kTcAPieceBytes /*r*/ +
                                kTcStages * kTcStageBytes + kTcStages * kTcYBytes + 256 /*barriers*/;

// ---- raw PTX wrappers ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tc_mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tc_mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "TC_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni TC_DONE;\n"
        "bra.uni TC_WAIT;\n"
        "TC_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tc_tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// the consumer warpgroups only (named barrier 1)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"r"(kTcConsumers) : "memory"); }

// shared-memory matrix descriptor of wgmma (cute::GMMA::GmmaDescriptor): start address, leading / stride byte offsets
// (all >> 4), layout type SWIZZLE_128B = 1 at bits 62..63
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) |
           (1ull << 62);
}

// D[64][64] (+)= A[64][16] . B[16][64], fp16 operands from shared memory, fp32 accumulators in registers.
// TRANS_B = 0: B is K-major ([n][k] in memory); 1: B is MN-major ([k][n]).  scale_d = 0 overwrites D.
// Accumulator layout (per thread of the warpgroup, warp w, lane l): d[4j + h] is row 16w + l/4 + 8 (h >> 1), column
// 8j + 2 (l % 4) + (h & 1).
template <int TRANS_B>
__device__ __forceinline__ void wg_mma_n64(float (&d)[32], uint64_t a_desc, uint64_t b_desc, int scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, %35;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a_desc), "l"(b_desc), "r"(scale_d), "n"(TRANS_B)
        : "memory");
}

// byte offset of element (row r, column k) of a [rows][128] fp16 tile stored as two [rows][64] blocks of block_bytes,
// rows 128 B apart, 16-byte chunks XOR-swizzled with the row (SWIZZLE_128B: what TMA writes and what wg_desc describes)
__device__ __forceinline__ uint32_t tc_tile_off(int r, int k, uint32_t block_bytes) {
    const int blk = k >> 6, kk = k & 63;
    return (uint32_t)(blk * block_bytes + r * 128 + ((((kk >> 3) ^ (r & 7)) << 4) | ((kk & 7) << 1)));
}

__device__ __forceinline__ float tc_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float tc_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float tc_lg2(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// The power-of-two exponent e that puts a row's (column's) largest magnitude m in [2^14, 2^15): every fp16 hi piece of
// v 2^e is finite and normal down to 2^-14 of m.  0 for an all-zero row; inf / NaN pass through unscaled.
__host__ __device__ __forceinline__ int tc_split_exponent(double m) {
    if (!(m > 0.0) || !(m < INFINITY)) return 0;
    int E;
    frexp(m, &E);  // m in [2^(E-1), 2^E)
    return 15 - E;
}

struct LogisticTcArgs {
    const float* y32;        // [n_slabs * 128] labels as fp32, zero padded
    long long N;             // true rows
    long long n_slabs;       // ceil(N / 128); X pieces are allocated with n_slabs * 128 rows (zero padded)
    const double* Q;         // [C][ldq] beta per chain
    long long ldq;
    const int* sx;           // [128] column exponents of the X pieces (X_k 2^sx[k])
    int C, K;
    double* Gpart;           // [gridDim.x][128 features][Cpad]  (feature-major)
    double* lpart;           // [gridDim.x][Cpad]
    int Cpad;
};

// 3 products x 8 k-steps of 16: hi*lo, lo*hi, then hi*hi.  a0/b0: shared addresses of the hi pieces; the lo pieces follow
// at +a_piece / +b_piece.  a_off / b_off give the byte offset of k-step ks inside a piece.
template <int TRANS_B, class AOff, class BOff>
__device__ __forceinline__ void tc_split_gemm(float (&d)[32], uint32_t a0, uint32_t a_piece, uint32_t b0, uint32_t b_piece,
                                              uint32_t b_lbo, AOff a_off, BOff b_off, bool accumulate) {
    int scale = accumulate ? 1 : 0;
#pragma unroll
    for (int prod = 0; prod < 3; ++prod) {
        const uint32_t a = a0 + (prod == 1 ? a_piece : 0u), b = b0 + (prod == 0 ? b_piece : 0u);
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            wg_mma_n64<TRANS_B>(d, wg_desc(a + a_off(ks), 16, 1024), wg_desc(b + b_off(ks), b_lbo, 1024), scale);
            scale = 1;
        }
    }
}

__global__ void __launch_bounds__(kTcThreads, 1)
    logistic_tc_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo, const LogisticTcArgs A) {
    extern __shared__ char tc_smem_raw[];
    char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
    char* beta_s = base;                                   // [hi | lo] pieces, 16 KB each
    char* r_s = beta_s + 2 * kTcAPieceBytes;               // [hi | lo] pieces of the residual tile, 16 KB each
    char* x_s = r_s + 2 * kTcAPieceBytes;                  // stages x [X_hi | X_lo]
    float* y_s = reinterpret_cast<float*>(x_s + kTcStages * kTcStageBytes);  // stages x [128] labels
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(y_s) + kTcStages * kTcYBytes);
    uint64_t* x_full = bars;          // [2] TMA -> consumers
    uint64_t* x_empty = bars + 2;     // [2] consumers (GEMM 2 done) -> TMA
    __shared__ double lp_wg_s[2][kTcChains];
    __shared__ float unscale_s[kTcChains];  // 2^-tau of each chain: eta = GEMM 1 accumulator * 2^-tau

    const int tid = threadIdx.x;
    const int c_base = blockIdx.y * kTcChains;
    // slabs of this CTA: blockIdx.x, blockIdx.x + gridDim.x, ...
    const long long my_slabs = (A.n_slabs > blockIdx.x) ? (A.n_slabs - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (tid == 0) {
        for (int i = 0; i < kTcStages; ++i) {
            mbar_init(&x_full[i], 1);
            mbar_init(&x_empty[i], kTcConsumers);
        }
    }
    // beta pieces.  Warp w stages chains w, w + 9, ... (lane: features lane + 32 j), four chains' loads in flight at a time:
    // beta_k 2^-sx[k] keeps eta = sum_k beta_k X_k, its per-chain maximum sets tau, and the fp16 hi / lo pieces of
    // beta_k 2^(tau - sx[k]) are written in the K-major SWIZZLE_128B image GEMM 1 reads as operand A
    constexpr int kWarps = kTcThreads / 32, kPer = 4;
    for (int c0 = tid >> 5; c0 < kTcChains; c0 += kPer * kWarps) {
        const int lane = tid & 31;
        double xs[4];  // 2^-sx[k] of this lane's features
#pragma unroll
        for (int j = 0; j < 4; ++j) xs[j] = ldexp(1.0, -A.sx[lane + 32 * j]);
        double v[kPer][4];
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            const int c = c0 + kWarps * i;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int k = lane + 32 * j;
                v[i][j] = (c < kTcChains && c_base + c < A.C && k < A.K) ? A.Q[(long long)(c_base + c) * A.ldq + k] * xs[j] : 0.0;
            }
        }
#pragma unroll
        for (int i = 0; i < kPer; ++i) {
            const int c = c0 + kWarps * i;
            double mx = fmax(fmax(fabs(v[i][0]), fabs(v[i][1])), fmax(fabs(v[i][2]), fabs(v[i][3])));
            for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(B200_FULL_MASK, mx, o));
            const int tau = tc_split_exponent(mx);
            if (c < kTcChains) {
                if (lane == 0) unscale_s[c] = ldexpf(1.0f, -tau);
                const double sc = ldexp(1.0, tau);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const double x = v[i][j] * sc;
                    const __half hi = __double2half(x);
                    const __half lo = __double2half(x - (double)__half2float(hi));
                    const uint32_t off = tc_tile_off(c, lane + 32 * j, kTcABlockBytes);
                    *reinterpret_cast<__half*>(beta_s + off) = hi;
                    *reinterpret_cast<__half*>(beta_s + kTcAPieceBytes + off) = lo;
                }
            }
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes of beta -> visible to wgmma
    __syncthreads();

    // warps 0..7: the two consumer warpgroups (wgmma needs warpgroup-aligned warps), warp 8: the producer
    if (tid >= kTcConsumers) {
        // ===== TMA producer: X_hi, X_lo (two 64-column boxes each) and the slab's labels =====
        if (tid == kTcConsumers) {
            for (long long s = 0; s < my_slabs; ++s) {
                const int st = (int)(s % kTcStages);
                if (s >= kTcStages) tc_mbar_wait(&x_empty[st], (uint32_t)(((s / kTcStages) - 1) & 1));
                const long long slab = blockIdx.x + s * gridDim.x;
                const int row0 = (int)(slab * kTcRows);
                char* dst = x_s + st * kTcStageBytes;
                mbar_expect_tx(&x_full[st], kTcStageBytes + kTcYBytes);
                tc_tma_load_2d(dst, &map_hi, 0, row0, &x_full[st]);
                tc_tma_load_2d(dst + kTcBlockBytes, &map_hi, 64, row0, &x_full[st]);
                tc_tma_load_2d(dst + kTcPieceBytes, &map_lo, 0, row0, &x_full[st]);
                tc_tma_load_2d(dst + kTcPieceBytes + kTcBlockBytes, &map_lo, 64, row0, &x_full[st]);
                tma_bulk_g2s(y_s + st * kTcRows, A.y32 + (long long)row0, kTcYBytes, &x_full[st]);
            }
        }
    } else {
        // ===== consumers: warpgroup wg owns slab rows 64 wg.. in GEMM 1 and features 64 wg.. in GEMM 2 =====
        const int t = tid, wg = t >> 7, wt = t & 127, warp = wt >> 5, lane = wt & 31;
        const int r0 = 16 * warp + (lane >> 2);        // chains r0 and r0 + 8 of this CTA
        const int col = 2 * (lane & 3);                // + 8 j + {0, 1}: column inside the warpgroup's 64
        const uint32_t beta_a = smem_u32(beta_s), r_a = smem_u32(r_s);
        double lp[2] = {0.0, 0.0};
        double gacc[32];  // fp64 gradient partials: d-layout of GEMM 2 (features 64 wg + 8j + col + {0,1}), all slabs
#pragma unroll
        for (int k = 0; k < 32; ++k) gacc[k] = 0.0;
        float g[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) g[k] = 0.0f;
        for (long long s = 0; s < my_slabs; ++s) {
            const int st = (int)(s % kTcStages);
            tc_mbar_wait(&x_full[st], (uint32_t)((s / kTcStages) & 1));
            const uint32_t xa = smem_u32(x_s + st * kTcStageBytes);
            // GEMM 1: eta for slab rows 64 wg .. 64 wg + 63 (row r of the slab is at r * 128 B inside each 64-column box)
            float eta[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) eta[k] = 0.0f;
            wg_fence();
            tc_split_gemm<0>(eta, beta_a, kTcAPieceBytes, xa + wg * 64 * 128, kTcPieceBytes, 16,
                             [](int ks) { return (uint32_t)((ks >> 2) * kTcABlockBytes + (ks & 3) * 32); },
                             [](int ks) { return (uint32_t)((ks >> 2) * kTcBlockBytes + (ks & 3) * 32); }, false);
            wg_commit();
            wg_wait_all();
            // residuals and log-likelihood terms
            const long long row_base = (blockIdx.x + s * gridDim.x) * kTcRows + 64 * wg;
            const float* ys = y_s + st * kTcRows + 64 * wg;
            float lp_s[2] = {0.f, 0.f};
            uint32_t rh[16], rl[16];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float rr[2];
#pragma unroll
                    for (int u = 0; u < 2; ++u) {
                        const int i = 8 * j + col + u;
                        const float x = eta[4 * j + 2 * hh + u] * unscale_s[r0 + 8 * hh];  // shared: no register held over the loop
                        const float yv = ys[i];
                        const float tt = tc_ex2(-1.4426950408889634f * fabsf(x));   // e^-|x|
                        const float w = 1.f + tt;
                        const float inv = tc_rcp(w);
                        const float sg = x >= 0.f ? inv : tt * inv;                  // sigmoid(x)
                        const float sp = fmaf(tc_lg2(w), 0.69314718055994530942f, fmaxf(x, 0.f));  // softplus(x)
                        // rows past N: X rows are zero (eta = 0), so the residual multiplies zero rows in GEMM 2
                        lp_s[hh] += (row_base + i < A.N) ? fmaf(yv, x, -sp) : 0.f;
                        rr[u] = yv - sg;
                    }
                    const __half2 h = __floats2half2_rn(rr[0], rr[1]);
                    const float2 hf = __half22float2(h);
                    const __half2 l = __floats2half2_rn(rr[0] - hf.x, rr[1] - hf.y);
                    rh[2 * j + hh] = *reinterpret_cast<const uint32_t*>(&h);
                    rl[2 * j + hh] = *reinterpret_cast<const uint32_t*>(&l);
                }
            }
            lp[0] += (double)lp_s[0];
            lp[1] += (double)lp_s[1];
            consumers_sync();  // both warpgroups are past GEMM 2 of the previous slab: the residual tile is free
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const uint32_t off = tc_tile_off(r0 + 8 * hh, 64 * wg + 8 * j + col, kTcABlockBytes);
                    *reinterpret_cast<uint32_t*>(r_s + off) = rh[2 * j + hh];
                    *reinterpret_cast<uint32_t*>(r_s + kTcAPieceBytes + off) = rl[2 * j + hh];
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            consumers_sync();  // the whole residual tile [64 chains][128 rows] is written
            // GEMM 2: g[c][k] += sum_i r[c][i] X[i][64 wg + k]; B = box wg of the stage, MN-major (16 rows = 2 KB per k-step)
            const bool first = (s % kTcDrain) == 0;
            wg_fence();
            tc_split_gemm<1>(g, r_a, kTcAPieceBytes, xa + wg * kTcBlockBytes, kTcPieceBytes, kTcBlockBytes,
                             [](int ks) { return (uint32_t)((ks >> 2) * kTcABlockBytes + (ks & 3) * 32); },
                             [](int ks) { return (uint32_t)(ks * 2048); }, !first);
            wg_commit();
            wg_wait_all();
            tc_mbar_arrive(&x_empty[st]);
            if ((s + 1) % kTcDrain == 0 || s + 1 == my_slabs) {
#pragma unroll
                for (int k = 0; k < 32; ++k) gacc[k] += (double)g[k];
            }
        }
        // row sums of the log-likelihood over the four lanes that share a chain (fixed order: deterministic)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            lp[hh] += __shfl_xor_sync(B200_FULL_MASK, lp[hh], 1);
            lp[hh] += __shfl_xor_sync(B200_FULL_MASK, lp[hh], 2);
        }
        if ((lane & 3) == 0) {
            lp_wg_s[wg][r0] = lp[0];
            lp_wg_s[wg][r0 + 8] = lp[1];
        }
        // the CTA's fp64 partial gradient, FEATURE-major [128 k][Cpad chains]
        double* gp = A.Gpart + (long long)blockIdx.x * kTcK * A.Cpad + c_base;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
            for (int h = 0; h < 4; ++h) {
                const int k = 64 * wg + 8 * j + col + (h & 1), c = r0 + 8 * (h >> 1);
                gp[(long long)k * A.Cpad + c] = gacc[4 * j + h];
            }
        }
        consumers_sync();
        if (t < kTcChains) A.lpart[(long long)blockIdx.x * A.Cpad + c_base + t] = lp_wg_s[0][t] + lp_wg_s[1][t];
    }
}

// labels as fp32, zero padded to whole slabs (copied into shared memory with the slab)
__global__ void __launch_bounds__(256) logistic_tc_y_kernel(const uint8_t* __restrict__ y, long long N, float* __restrict__ y32,
                                                            long long rows_pad) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < rows_pad) y32[e] = (e < N) ? (float)y[e] : 0.f;
}

// colmax[k] = max_i |X[i][k]| over the N rows and K columns of the fp64 design matrix (row stride ldx), 0 for k >= K;
// colmax[128] zeroed by the caller.  The bit patterns of non-negative doubles order like their values: the result does not
// depend on the order of the atomics.
__global__ void __launch_bounds__(256) logistic_tc_colmax_kernel(const double* __restrict__ X, long long N, int K, long long ldx,
                                                                 unsigned long long* __restrict__ colmax) {
    const int k = threadIdx.x & 127;
    double m = 0.0;
    if (k < K)
        for (long long r = 2LL * blockIdx.x + (threadIdx.x >> 7); r < N; r += 2LL * gridDim.x) m = fmax(m, fabs(X[r * ldx + k]));
    atomicMax(colmax + k, (unsigned long long)__double_as_longlong(m));
}

__global__ void tc_exponent_kernel(const unsigned long long* __restrict__ mx, int n, int* __restrict__ e) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) e[i] = tc_split_exponent(__longlong_as_double((long long)mx[i]));
}

// fp64 design matrix [N][K] (row stride ldx) -> fp16 pieces of X_k 2^sx[k], [n_slabs * 128][128], zero padded
__global__ void __launch_bounds__(256) logistic_tc_split_kernel(const double* __restrict__ X, long long N, int K, long long ldx,
                                                                const int* __restrict__ sx, __half* __restrict__ Xh,
                                                                __half* __restrict__ Xl, long long rows_pad) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows_pad * kTcK) return;
    const long long r = e >> 7;
    const int k = (int)(e & 127);
    const double v = (r < N && k < K) ? ldexp(X[r * ldx + k], sx[k]) : 0.0;
    const __half hi = __double2half(v);
    Xh[e] = hi;
    Xl[e] = __double2half(v - (double)__half2float(hi));
}

}  // namespace b200
