// D[c][j] = alpha * sum_k A[c][k] * B[j][k]  on the Hopper tensor cores (wgmma.mma_async, TMA): the PERFORMANCE mode of
// the dense Gaussian config (BASELINE #5: grad = -P q, w = Sigma g, p0 = L^-T z, v0 = L z at n = 10^4).  Same arithmetic
// as csrc/logistic_tc.cuh: every fp64 operand is hi + lo in fp16 (22 significant bits), a product is hi*hi + hi*lo + lo*hi
// in three f16 MMAs with fp32 accumulation, and the fp32 accumulator only ever covers one k-block (64 terms) before it is
// drained into compensated fp32 register sums (kahan_add).  The fp64 DMMA kernel of dense.cuh stays the parity mode.
//
// B (the model's n x n matrices) is split once at b200_model_set_precision; A (the chains' vectors) is split by
// gemm_tc_split_kernel before every GEMM.  Each row is first scaled by an exact power of two that puts its maximum in
// [2^14, 2^15) (tc_split_exponent: fp16 keeps 2^-14 .. 65504 only): eb[j] for row j of B, once; ea[c] for row c of A, found
// by the split kernel itself (one CTA per row: row maximum, then the pieces) before every GEMM.  The epilogue multiplies
// by 2^-(ea[c] + eb[j]), so the result does not depend on the scale of the data.  Both are K-major fp16 [rows][Kpad] in HBM, TMA-loaded in 64-wide k-blocks with
// SWIZZLE_128B.  CTA tile = 128 chains x 64 outputs: two consumer warpgroups (64 chains each, sharing
// the B tile) and a producer warp; tiles are walked output-block-major so that the chain tiles of one output block run together and share B
// through L2.
#pragma once
#include "logistic_tc.cuh"

namespace b200 {

constexpr int kGtM = 128;        // chains per tile (two warpgroups of 64)
constexpr int kGtN = 64;         // outputs per tile
constexpr int kGtKB = 64;        // k per block (128 B of fp16: one swizzle row)
constexpr int kGtStages = 4;
constexpr int kGtConsumers = 256;
constexpr int kGtThreads = 32 + kGtConsumers;
constexpr uint32_t kGtABytes = kGtM * kGtKB * 2;                    // 16 KB per piece
constexpr uint32_t kGtBBytes = kGtN * kGtKB * 2;                    // 8 KB per piece
constexpr uint32_t kGtStageBytes = 2 * kGtABytes + 2 * kGtBBytes;   // 48 KB
constexpr size_t kGtSmemBytes = 1024 + (size_t)kGtStages * kGtStageBytes + 256;

// Compensated (Kahan) fp32 accumulation of one drained value: s + (-c) carries the running sum to ~2^-24 of its magnitude
// independently of the number of terms.
__device__ __forceinline__ void kahan_add(float& s, float& c, float x) {
    const float y = x - c;
    const float t = s + y;
    c = (t - s) - y;
    s = t;
}

// 2^e as a double, exactly (a multiply by it is ldexp); a few integer instructions in the normal range instead of ldexp's
// general path, which matters in an epilogue that runs once per output
__device__ __forceinline__ double tc_pow2(int e) {
    return (e >= -1022 && e <= 1023) ? __longlong_as_double((long long)(e + 1023) << 52) : ldexp(1.0, e);
}

struct GemmTcArgs {
    int C, Nout, n_kblocks;   // chains, outputs, k-blocks of 64 (operands are zero padded to that)
    double alpha;
    double* D;                // [C][ldd]
    long long ldd;
    const int* ea;            // [C] row exponents of the A pieces (A_c 2^ea[c])
    const int* eb;            // [Nout] row exponents of the B pieces
    int n_tiles_m, n_tiles;   // chain tiles per output block, total tiles
};

__global__ void __launch_bounds__(kGtThreads, 1)
    gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                   const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo, const GemmTcArgs G) {
    extern __shared__ char gt_smem_raw[];
    char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(gt_smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + kGtStages * kGtStageBytes);
    uint64_t* full = bars;                 // [stages] TMA -> consumers
    uint64_t* empty = bars + kGtStages;    // [stages] consumers -> TMA
    const int tid = threadIdx.x;
    const int KB = G.n_kblocks;

    if (tid == 0) {
        for (int i = 0; i < kGtStages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], kGtConsumers);
        }
    }
    __syncthreads();

    // warps 0..7: the two consumer warpgroups (wgmma needs warpgroup-aligned warps), warp 8: the producer
    if (tid >= kGtConsumers) {
        if (tid == kGtConsumers) {
            long long it = 0;  // k-blocks loaded so far (over all tiles of this CTA)
            for (int tile = blockIdx.x; tile < G.n_tiles; tile += gridDim.x) {
                const int c0 = (tile % G.n_tiles_m) * kGtM, j0 = (tile / G.n_tiles_m) * kGtN;
                for (int kb = 0; kb < KB; ++kb, ++it) {
                    const int st = (int)(it % kGtStages);
                    if (it >= kGtStages) tc_mbar_wait(&empty[st], (uint32_t)(((it / kGtStages) - 1) & 1));
                    char* dst = base + st * kGtStageBytes;
                    mbar_expect_tx(&full[st], kGtStageBytes);
                    tc_tma_load_2d(dst, &map_a_hi, kb * kGtKB, c0, &full[st]);
                    tc_tma_load_2d(dst + kGtABytes, &map_a_lo, kb * kGtKB, c0, &full[st]);
                    tc_tma_load_2d(dst + 2 * kGtABytes, &map_b_hi, kb * kGtKB, j0, &full[st]);
                    tc_tma_load_2d(dst + 2 * kGtABytes + kGtBBytes, &map_b_lo, kb * kGtKB, j0, &full[st]);
                }
            }
        }
    } else {
        // consumers: warpgroup wg owns chains 64 wg .. 64 wg + 63 of the tile
        const int wg = tid >> 7, wt = tid & 127, warp = wt >> 5, lane = wt & 31;
        const int r0 = 16 * warp + (lane >> 2), col = 2 * (lane & 3);
        long long it = 0;
        for (int tile = blockIdx.x; tile < G.n_tiles; tile += gridDim.x) {
            const int c0 = (tile % G.n_tiles_m) * kGtM + 64 * wg, j0 = (tile / G.n_tiles_m) * kGtN;
            float sum[32], comp[32];
#pragma unroll
            for (int k = 0; k < 32; ++k) { sum[k] = 0.0f; comp[k] = 0.0f; }
            for (int kb = 0; kb < KB; ++kb, ++it) {
                const int st = (int)(it % kGtStages);
                tc_mbar_wait(&full[st], (uint32_t)((it / kGtStages) & 1));
                const uint32_t a_hi = smem_u32(base + st * kGtStageBytes) + wg * 64 * 128;
                const uint32_t b_hi = smem_u32(base + st * kGtStageBytes) + 2 * kGtABytes;
                float d[32];
#pragma unroll
                for (int k = 0; k < 32; ++k) d[k] = 0.0f;
                wg_fence();
                int scale = 0;
#pragma unroll
                for (int prod = 0; prod < 3; ++prod) {  // hi*lo, lo*hi, then hi*hi (small products first)
                    const uint32_t a = a_hi + (prod == 1 ? kGtABytes : 0u), b = b_hi + (prod == 0 ? kGtBBytes : 0u);
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        wg_mma_n64<0>(d, wg_desc(a + ks * 32, 16, 1024), wg_desc(b + ks * 32, 16, 1024), scale);
                        scale = 1;
                    }
                }
                wg_commit();
                wg_wait_all();
                tc_mbar_arrive(&empty[st]);
#pragma unroll
                for (int k = 0; k < 32; ++k) kahan_add(sum[k], comp[k], d[k]);
            }
            // the row exponents of this thread's 2 chains and 16 outputs, loaded before any store (D may alias them as far as
            // the compiler knows, which would serialise one load round trip per stored element)
            int ea[2], eb[16];
#pragma unroll
            for (int h = 0; h < 2; ++h) ea[h] = (c0 + r0 + 8 * h < G.C) ? G.ea[c0 + r0 + 8 * h] : 0;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int jj = j0 + 8 * (j >> 1) + col + (j & 1);
                eb[j] = (jj < G.Nout) ? G.eb[jj] : 0;
            }
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int h = 0; h < 4; ++h) {
                    const int c = c0 + r0 + 8 * (h >> 1), jj = j0 + 8 * j + col + (h & 1);
                    if (c < G.C && jj < G.Nout)
                        G.D[(long long)c * G.ldd + jj] =
                            G.alpha * (((double)sum[4 * j + h] - (double)comp[4 * j + h]) * tc_pow2(-(ea[h >> 1] + eb[2 * j + (h & 1)])));
                }
            }
        }
    }
}

// fp64 [rows][ld] (first `cols` columns) -> fp16 pieces of row r times 2^e_row[r], [rows_pad][kpad], zero padded, and
// e_row[r] = tc_split_exponent(max_k |X[r][k]|) (0 for rows .. rows_pad).  One CTA of kGtSplitThreads threads per row: the row
// maximum first, then the pieces from the same row, now in L1 / L2 (a row of 10^4 doubles is 10 elements per thread).
constexpr int kGtSplitThreads = 1024;
__global__ void __launch_bounds__(kGtSplitThreads) gemm_tc_split_kernel(const double* __restrict__ X, long long rows, long long cols,
                                                                        long long ld, int* __restrict__ e_row, __half* __restrict__ Xh,
                                                                        __half* __restrict__ Xl, long long kpad) {
    __shared__ double wmax[kGtSplitThreads / 32];
    const long long r = blockIdx.x;
    const double* x = X + r * ld;
    double m = 0.0;
    if (r < rows) {
#pragma unroll 4
        for (long long k = threadIdx.x; k < cols; k += kGtSplitThreads) m = fmax(m, fabs(x[k]));
    }
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(B200_FULL_MASK, m, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kGtSplitThreads / 32; ++w) m = fmax(m, wmax[w]);
    const int es = tc_split_exponent(m);
    if (threadIdx.x == 0) e_row[r] = es;
    const double sc = ldexp(1.0, es);  // exact scaling: every scaled entry is <= 2^15
#pragma unroll 4
    for (long long k = threadIdx.x; k < kpad; k += kGtSplitThreads) {
        const double v = (r < rows && k < cols) ? x[k] * sc : 0.0;
        const __half hi = __double2half(v);
        Xh[r * kpad + k] = hi;
        Xl[r * kpad + k] = __double2half(v - (double)__half2float(hi));
    }
}

}  // namespace b200
