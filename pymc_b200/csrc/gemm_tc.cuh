// D[c][j] = alpha * sum_k A[c][k] * B[j][k]  on the Hopper tensor cores (wgmma.mma_async, TMA): the PERFORMANCE mode of
// the dense Gaussian config (BASELINE #5: grad = -P q, w = Sigma g, p0 = L^-T z, v0 = L z at n = 10^4).  Same arithmetic
// as csrc/logistic_tc.cuh: every fp64 operand is hi + lo in fp16 (22 significant bits), a product is hi*hi + hi*lo + lo*hi
// in three f16 MMAs with fp32 accumulation, and the fp32 accumulator only ever covers one k-block (64 terms) before it is
// drained into compensated fp32 register sums (kahan_add).  The fp64 DMMA kernel of dense.cuh stays the parity mode.
//
// B (the model's n x n matrices) is split once at b200_model_set_precision; A (the chains' vectors) is split by
// gemm_tc_split_kernel before every GEMM.  Both are K-major fp16 [rows][Kpad] in HBM, TMA-loaded in 64-wide k-blocks with
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

struct GemmTcArgs {
    int C, Nout, n_kblocks;   // chains, outputs, k-blocks of 64 (operands are zero padded to that)
    double alpha;
    double* D;                // [C][ldd]
    long long ldd;
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
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int h = 0; h < 4; ++h) {
                    const int c = c0 + r0 + 8 * (h >> 1), jj = j0 + 8 * j + col + (h & 1);
                    if (c < G.C && jj < G.Nout)
                        G.D[(long long)c * G.ldd + jj] = G.alpha * ((double)sum[4 * j + h] - (double)comp[4 * j + h]);
                }
            }
        }
    }
}

// fp64 [rows][ld] (first `cols` columns) -> fp16 pieces [rows_pad][kpad], zero padded
__global__ void __launch_bounds__(256) gemm_tc_split_kernel(const double* __restrict__ X, long long rows, long long cols, long long ld,
                                                            __half* __restrict__ Xh, __half* __restrict__ Xl, long long rows_pad,
                                                            long long kpad) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows_pad * kpad) return;
    const long long r = e / kpad, k = e % kpad;
    const double v = (r < rows && k < cols) ? X[r * ld + k] : 0.0;
    const __half hi = __double2half(v);
    Xh[e] = hi;
    Xl[e] = __double2half(v - (double)__half2float(hi));
}

}  // namespace b200
