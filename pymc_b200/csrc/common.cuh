// Shared device helpers: team (warp / block) reductions, libm-shaped scalar functions, bulk-TMA staging.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/b200nuts.h"

#define B200_FULL_MASK 0xffffffffu

#define B200_HALF_LOG_2PI 0.91893853320467274178032973640562

namespace b200 {

// ---------------------------------------------------------------------------------------------
// scalar helpers (same branch structure as the NumPy functions the reference calls)
// ---------------------------------------------------------------------------------------------
// log(1 + x) for x >= 0 where the result is ADDED to an O(1) or larger log-density / log-weight: forming 1 + x first costs
// at most 1.1e-16 ABSOLUTE error, invisible next to the terms it is added to, at half the instructions of log1p().
__device__ __forceinline__ double log1p_abs(double x) { return log(1.0 + x); }

// numpy.logaddexp (npy_logaddexp): used at hmc/nuts.py:415,376,465
__device__ __forceinline__ double logaddexp(double x, double y) {
    if (x == y) return x + 0.69314718055994530942;  // log 2
    const double d = x - y;
    if (d > 0) return x + log1p(exp(-d));
    if (d <= 0) return y + log1p(exp(d));
    return x + y;  // NaN
}

__device__ __forceinline__ double softplus(double x) {
    return fmax(x, 0.0) + log1p(exp(-fabs(x)));
}

__device__ __forceinline__ double sigmoid(double x) {
    const double e = exp(-fabs(x));
    const double r = 1.0 / (1.0 + e);
    return x >= 0 ? r : e * r;
}

// digamma psi(x) for x > 0 (CUDA's libm has none): the upward recurrence psi(x) = psi(x + 1) - 1/x up to x >= 10, then the
// asymptotic series log x - 1/(2x) - sum_k B_2k / (2k x^2k) through x^-14, whose truncation error at x = 10 is below 1e-16.
__device__ __forceinline__ double digamma(double x) {
    double acc = 0.0;
    while (x < 10.0) {
        acc -= 1.0 / x;
        x += 1.0;
    }
    const double r = 1.0 / x, r2 = r * r;
    const double ser =
        r2 * (1.0 / 12 - r2 * (1.0 / 120 - r2 * (1.0 / 252 - r2 * (1.0 / 240 - r2 * (1.0 / 132 - r2 * (691.0 / 32760 - r2 / 12.0))))));
    return acc + log(x) - 0.5 * r - ser;
}

// Normal(0,1) log-density constant part is added by callers; this is the HalfCauchy(beta) density of
// x = exp(z) plus the log-transform Jacobian (+z), and its derivative in z.
// Reference: Cauchy.logp continuous.py:2287-2288, HalfCauchy.logp :2383-2385, LogTransform
// logprob/transforms.py:880-891.  `x` must be exp(z) (passed in so callers can share the exp).
__device__ __forceinline__ void halfcauchy_log(double z, double x, double beta, double log_beta,
                                               double& val, double& dz) {
    const double t = x * (1.0 / beta);
    // rounded product: an unmarked t * t lets ptxas fuse it into 1 + t * t below at some inlining sites and not at others
    // (it did so in the batched Eight Schools logp kernel but not in its NUTS kernel), so one model's logp at one point
    // would differ between kernels by an ulp
    const double u = __dmul_rn(t, t);
    val = (0.69314718055994530942 - 1.1447298858494001741 /* log pi */) - log_beta - log1p_abs(u) + z;
    dz = 1.0 - 2.0 * u / (1.0 + u);
}

// ---------------------------------------------------------------------------------------------
// Warp team: one chain = one warp; lane l owns elements l, l+32, ...  All reductions are xor
// butterflies, so every lane ends with bit-identical results (commutativity of IEEE add) and all
// tree decisions are warp-uniform without a broadcast.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(B200_FULL_MASK, x, o);
    return x;
}

template <int N>
__device__ __forceinline__ void warp_sum_n(double (&x)[N]) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int i = 0; i < N; ++i) x[i] += __shfl_xor_sync(B200_FULL_MASK, x[i], o);
    }
}

// All-reduce of N <= 8 values in 9 + N double-shuffles instead of 5 N: a reduce-scatter over lane bits
// 4,3,2 (each step halves the values a lane carries), a butterfly over bits 1,0, then one broadcast per
// value.  Every lane receives the broadcast of the same lane's total, so results are warp-uniform bits.
template <int N>
__device__ __forceinline__ void warp_sum_bcast_n(double (&x)[N], int lane) {
    static_assert(N >= 1 && N <= 8, "warp_sum_bcast_n handles up to 8 values");
    double v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (i < N) ? x[i] : 0.0;
    double w[4], u[2];
    {
        const bool up = lane & 16;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const double send = up ? v[i] : v[i + 4], keep = up ? v[i + 4] : v[i];
            w[i] = keep + __shfl_xor_sync(B200_FULL_MASK, send, 16);
        }
    }
    {
        const bool up = lane & 8;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const double send = up ? w[i] : w[i + 2], keep = up ? w[i + 2] : w[i];
            u[i] = keep + __shfl_xor_sync(B200_FULL_MASK, send, 8);
        }
    }
    double t;
    {
        const bool up = lane & 4;
        const double send = up ? u[0] : u[1], keep = up ? u[1] : u[0];
        t = keep + __shfl_xor_sync(B200_FULL_MASK, send, 4);
    }
    t += __shfl_xor_sync(B200_FULL_MASK, t, 2);
    t += __shfl_xor_sync(B200_FULL_MASK, t, 1);
    // lane holds the total of value j = 4*bit4 + 2*bit3 + bit2
#pragma unroll
    for (int j = 0; j < N; ++j)
        x[j] = __shfl_sync(B200_FULL_MASK, t, ((j & 4) ? 16 : 0) | ((j & 2) ? 8 : 0) | ((j & 1) ? 4 : 0));
}

// ---------------------------------------------------------------------------------------------
// Team = the W warps that own one chain (W = 1: a warp, several chains per CTA; W > 1: the whole CTA).
// Thread t of the team owns elements t, t + 32W, ...  Cross-warp reductions go through `red`
// (W x 8 doubles of shared memory) in a fixed order, so all threads of the team get identical bits.
// ---------------------------------------------------------------------------------------------
template <int W>
__device__ __forceinline__ void team_sync() {
    if constexpr (W == 1) __syncwarp(); else __syncthreads();
}

template <int W, int N>
__device__ __forceinline__ void team_sum_n(double (&x)[N], int tid, double* red) {
    static_assert(N <= 8, "team_sum_n handles up to 8 values");
    if constexpr (W == 1) {
        if constexpr (N >= 4) warp_sum_bcast_n(x, tid); else warp_sum_n(x);
    } else {
        warp_sum_n(x);
        const int w = tid >> 5;
        if ((tid & 31) == 0) {
#pragma unroll
            for (int i = 0; i < N; ++i) red[w * 8 + i] = x[i];
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < N; ++i) {
            double a = red[i];
#pragma unroll
            for (int ww = 1; ww < W; ++ww) a += red[ww * 8 + i];
            x[i] = a;
        }
        __syncthreads();
    }
}

template <int W>
__device__ __forceinline__ double team_sum(double x, int tid, double* red) {
    double a[1] = {x};
    team_sum_n<W>(a, tid, red);
    return a[0];
}

// ---------------------------------------------------------------------------------------------
// Bulk TMA (cp.async.bulk, SASS UBLKCP): stage a contiguous global array into shared memory,
// completion signalled on an mbarrier.  bytes must be a multiple of 16, both addresses 16B aligned.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}

__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                             uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(phase)
        : "memory");
}

// Draw post-processing fused into the record step (SURVEY 8f-1): the backward transform of one element, what the reference
// evaluates per draw through a compiled function (backends/ndarray.py:108; transforms logprob/transforms.py:880-891,
// :1026-1045).  kind == null: the unconstrained value is recorded.
__device__ __forceinline__ double constrained(double q, int i, const signed char* kind, const double* lo, const double* hi) {
    if (!kind) return q;
    const int t = kind[i];
    if (t == 1) return exp(q);
    if (t == 2) {
        const double s = sigmoid(q);
        return s * hi[i] + (1.0 - s) * lo[i];
    }
    return q;
}

}  // namespace b200
