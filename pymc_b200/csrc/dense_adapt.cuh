// Per-chain adaptive dense mass matrix for the lock-step engine: QuadPotentialFullAdapt (hmc/quadpotential.py:748-845) with
// its two _WeightedCovariance estimators (:855-907) -- init="adapt_full" / "jitter+adapt_full" (sampling/mcmc.py:1986-2005).
//
// Every chain owns four n x n matrices in HBM (row-major, no padding): the covariance `_cov`, its lower Cholesky factor
// `_chol`, and the raw scatter matrices of the foreground and background estimators.  The lock-step advance kernel
// (lockstep.cuh) stops a chain at the end of a draw (phase 3); between two advance calls
//     fa_update_momentum_kernel   potential.update(sample, grad, tune)  -> add_sample x 2, current_covariance, Cholesky,
//                                 window switch (:818-843); then potential.random() of the next draw:
//                                 p0 = solve_triangular(chol^T, z) (:710-713) and v0 = cov p0 (:705-707, integration.py:72)
//     fa_symv_kernel              w = cov g for every requested point (the per-chain form of the mass GEMM)
// run for the chains that asked.  One CTA per chain.  The estimator arithmetic is NumPy's (unfused elementwise products and
// sums, IEEE division), so `_cov` equals the reference's bit for bit while the draws do; the Cholesky factorisation, the
// triangular solve and the matrix-vector products sum in their own order (LAPACK's / BLAS's orders are implementation
// details), which is why parity for this potential is stated to a tolerance (tests/test_gpu_dense_adapt.py).
#pragma once
#include "lockstep.cuh"

namespace b200 {

constexpr int kFaThreads = 256;
constexpr int kFaMaxN = 1024;  // five n-vectors of shared memory per CTA; the matrices are 4 n^2 doubles per chain
__host__ __device__ inline size_t fa_smem_bytes(int n) { return (size_t)5 * n * sizeof(double); }

// initial state of the matrices: cov = diag(var0) (identity when var0 is null), chol = diag(sqrt(var0)),
// foreground raw = cov * initial_weight, background raw = eye * 0 (quadpotential.py:803-808, :876-885)
__global__ void __launch_bounds__(kFaThreads) fa_init_kernel(const LsDev P) {
    const int chain = blockIdx.x, n = P.n;
    const long long nn = (long long)n * n;
    double* cov = P.fa_cov + chain * nn;
    double* chol = P.fa_chol + chain * nn;
    double* fg = P.fa_raw + (2LL * chain + 0) * nn;
    double* bg = P.fa_raw + (2LL * chain + 1) * nn;
    for (long long idx = threadIdx.x; idx < nn; idx += blockDim.x) {
        const int i = (int)(idx / n), j = (int)(idx - (long long)i * n);
        const double v = (i == j) ? (P.var0 ? P.var0[(long long)chain * n + i] : 1.0) : 0.0;
        cov[idx] = v;
        chol[idx] = (i == j) ? sqrt(v) : 0.0;
        fg[idx] = v * P.init_weight;
        bg[idx] = 0.0;
    }
}

// out[i] = sum_j M[i][j] x[j]; x in shared memory; one warp per row, lanes stride the row (coalesced), xor-butterfly sum
__device__ __forceinline__ void fa_matvec(const double* __restrict__ M, const double* x_s, double* out, int n) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int i = w; i < n; i += nw) {
        const double* row = M + (long long)i * n;
        double s0 = 0.0, s1 = 0.0;
        int j = lane;
        for (; j + 32 < n; j += 64) { s0 = fma(row[j], x_s[j], s0); s1 = fma(row[j + 32], x_s[j + 32], s1); }
        if (j < n) s0 = fma(row[j], x_s[j], s0);
        const double s = warp_sum(s0 + s1);
        if (lane == 0) out[i] = s;
    }
}

// w = cov_c g for the point every live chain asked for (QuadPotentialFull.velocity, quadpotential.py:705-707)
__global__ void __launch_bounds__(kFaThreads) fa_symv_kernel(const LsDev P) {
    extern __shared__ double fa_s[];
    const int chain = blockIdx.x, n = P.n;
    const int phase = P.state[chain].phase;
    if (phase != 0 && phase != 1) return;  // finished chains have given their row up; phase-3 chains wait for momentum
    const int row = P.slot ? P.slot[chain] : chain;
    const double* g = P.Greq + (long long)row * P.ld;
    for (int i = threadIdx.x; i < n; i += blockDim.x) fa_s[i] = g[i];
    __syncthreads();
    fa_matvec(P.fa_cov + (long long)chain * n * n, fa_s, P.Wreq + (long long)row * P.ld, n);
}

// Lower Cholesky factor of A (lower triangle read) into Lo, right-looking, column k staged in shared memory.
// Returns false (uniformly) when a pivot is not positive (scipy.linalg.cholesky raises LinAlgError).
__device__ bool fa_cholesky(const double* __restrict__ A, double* Lo, double* col_s, int n) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const long long nn = (long long)n * n;
    for (long long idx = threadIdx.x; idx < nn; idx += blockDim.x) {
        const int i = (int)(idx / n), j = (int)(idx - (long long)i * n);
        Lo[idx] = (j <= i) ? A[idx] : 0.0;
    }
    __syncthreads();
    for (int k = 0; k < n; ++k) {
        const double d = Lo[(long long)k * n + k];
        if (!(d > 0.0)) return false;  // every thread reads the same value: uniform exit
        const double r = sqrt(d);
        for (int i = k + 1 + (int)threadIdx.x; i < n; i += blockDim.x) {
            const double v = Lo[(long long)i * n + k] / r;
            Lo[(long long)i * n + k] = v;
            col_s[i] = v;
        }
        __syncthreads();  // also orders every thread's read of the pivot before its overwrite
        if (threadIdx.x == 0) Lo[(long long)k * n + k] = r;
        for (int i = k + 1 + w; i < n; i += nw) {
            const double ci = col_s[i];
            double* row = Lo + (long long)i * n;
            for (int j = k + 1 + lane; j <= i; j += 32) row[j] = fma(-ci, col_s[j], row[j]);
        }
        __syncthreads();
    }
    return true;
}

__global__ void __launch_bounds__(kFaThreads) fa_update_momentum_kernel(const LsDev P, int m) {
    extern __shared__ double fa_s[];
    const int jj = blockIdx.x;
    if (jj >= m) return;
    const int chain = P.mom_list[jj], n = P.n, tid = threadIdx.x;
    const long long nn = (long long)n * n;
    LsState* SP = P.state + chain;
    // scalars of the chain (identical in every thread; thread 0 writes them back).  Only the window's mean slots are used:
    // dw.swap() also exchanges the variance slot ids, which nothing reads under DENSE_ADAPT.
    DiagWindow dw = SP->dw;
    int prev = SP->prev_update, fa_fg = SP->fa_fg;
    const int upd = SP->upd_pending, it = SP->mom_it;
    int chol_bad = SP->chol_bad;
    double* vb = P.vecs + (long long)chain * P.vec_stride;
    double* cov = P.fa_cov + chain * nn;
    double* chol = P.fa_chol + chain * nn;
    double* before_f = fa_s, *after_f = fa_s + n, *before_b = fa_s + 2 * n, *after_b = fa_s + 3 * n, *tmp = fa_s + 4 * n;

    if (upd) {
        // ---- QuadPotentialFullAdapt.update (quadpotential.py:818-843), sample = the accepted position ------------------
        const int delta = dw.k_samples - prev;
        const double* x = vb + (long long)LV_Q * n;
        double* fm = vb + (long long)dw.fg_m * n;
        double* bm = vb + (long long)dw.bg_m * n;
        dw.fg_n += 1.0; dw.bg_n += 1.0;  // _WeightedCovariance.add_sample :887-893
        for (int i = tid; i < n; i += blockDim.x) {
            const double xi = x[i];
            before_f[i] = welford_mean(xi, dw.fg_n, fm[i]); after_f[i] = xi - fm[i];
            before_b[i] = welford_mean(xi, dw.bg_n, bm[i]); after_b[i] = xi - bm[i];
        }
        __syncthreads();
        const bool refresh = ((delta + 1) % P.upd_window) == 0;
        double* F = P.fa_raw + (2LL * chain + fa_fg) * nn;
        double* B = P.fa_raw + (2LL * chain + (fa_fg ^ 1)) * nn;
        const double denom = dw.fg_n - 1.0;  // current_covariance :895-901
        for (long long idx = tid; idx < nn; idx += blockDim.x) {
            const int i = (int)(idx / n), j = (int)(idx - (long long)i * n);
            const double f = __dadd_rn(F[idx], __dmul_rn(after_f[i], before_f[j]));
            F[idx] = f;
            B[idx] = __dadd_rn(B[idx], __dmul_rn(after_b[i], before_b[j]));
            if (refresh) cov[idx] = f / denom;
        }
        __syncthreads();
        if (refresh) {
            // _update_from_weightvar :810-816: a failed factorisation keeps the old factor and is reported (raise_ok)
            if (!fa_cholesky(cov, chol, tmp, n)) chol_bad = 1;  // (the frozen chain never reads the half-written factor)
            __syncthreads();
            // the chain state's w = cov . grad follows the new covariance
            const double* g = vb + (long long)LV_G * n;
            for (int i = tid; i < n; i += blockDim.x) tmp[i] = g[i];
            __syncthreads();
            fa_matvec(cov, tmp, vb + (long long)LV_W * n, n);
            __syncthreads();
        }
        if (delta >= dw.window) {  // the background estimator takes over; a fresh one starts (:833-841)
            fa_fg ^= 1;
            dw.swap();
            double* nb = P.fa_raw + (2LL * chain + (fa_fg ^ 1)) * nn;
            for (long long idx = tid; idx < nn; idx += blockDim.x) nb[idx] = 0.0;  // eye * n_samples(0)
            double* nm = vb + (long long)dw.bg_m * n;
            for (int i = tid; i < n; i += blockDim.x) nm[i] = 0.0;
            prev = dw.k_samples;
            dw.window = (int)(dw.window * P.win_mult);
        }
        ++dw.k_samples;
    }

    // ---- potential.random() for draw `it`: p0 = solve_triangular(chol^T, z) (quadpotential.py:710-713) ---------------------
    double* b = before_f;   // right-hand side, updated in place
    double* px = after_f;   // solution
    for (int i = tid; i < n; i += blockDim.x) b[i] = momentum_z(P, chain, it, i);
    __syncthreads();
    for (int j = n - 1; j >= 0; --j) {  // back substitution, row j of the factor is column j of its transpose (contiguous)
        const double* Lj = chol + (long long)j * n;
        const double xj = b[j] / Lj[j];
        if (tid == 0) px[j] = xj;
        for (int i = tid; i < j; i += blockDim.x) b[i] = fma(-Lj[i], xj, b[i]);
        __syncthreads();
    }
    double* p0 = P.P0n + (long long)chain * P.ld;
    for (int i = tid; i < n; i += blockDim.x) p0[i] = px[i];
    // v0 = cov p0 (QuadPotentialFull.velocity at compute_state, integration.py:72)
    fa_matvec(cov, px, P.V0n + (long long)chain * P.ld, n);

    if (tid == 0) {
        SP->dw = dw; SP->prev_update = prev; SP->fa_fg = fa_fg; SP->upd_pending = 0; SP->chol_bad = chol_bad;
        SP->mom_have = it;
    }
}

}  // namespace b200
