// The per-draw bookkeeping that the persistent engine (nuts_warp.cuh) and the lock-step engine (lockstep.cuh) share: the run
// configuration, dual-averaging step size, diagonal Welford windows, the 12 per-draw statistics, frozen-chain outputs, the
// chain summary and the momentum noise.  Tree building differs between the engines (registers and shared memory vs HBM
// vectors); everything here is written once so that a fix to an adaptation rule or a statistic cannot miss an engine.
//
// The persistent kernel has no register headroom: every function is force-inlined and the state structs are plain scalars,
// which the compiler splits into registers like the loose locals they replace.
#pragma once
#include "../../include/b200nuts.h"
#include "common.cuh"
#include "rng.cuh"

namespace b200 {

// What both engines read of a b200_nuts_run call: sizes, schedule, adaptation constants, inputs and outputs.
struct RunCfg {
    int C, n, tune, draws, max_td, early_td, adapt_step, mass_kind, momentum_source, store_warmup;
    int window, discard, chain_offset;
    int it0, n_iter;                           // this call runs the iterations [it0, it0 + n_iter) of the chain's schedule
    double eps0, target, gamma, kappa, t0, Emax, init_weight;
    unsigned long long philox_seed;
    const double* q0;     // [C][n]
    const double* var0;   // [C][n] or null
    const double* mean0;  // [C][n] or null
    const double* eps0c;  // [C] or null: per-chain initial step size
    const double* z;      // [C][n_iter][n] or null
    b200_pcg64* rng;      // [C]
    double* draws_out;    // [C][T][n]
    const signed char* tr_kind;  // [n] or null: record CONSTRAINED values (0 identity, 1 exp, 2 lo + (hi - lo) sigmoid)
    const double* tr_lo;         // [n]
    const double* tr_hi;         // [n]
    b200_stats st;
    b200_chain_summary sm;
};

// DualAverageAdaptation (step_sizes.py:41-84); products and sums kept unfused like the Python scalars
struct StepSize {
    double log_step, log_bar, hbar, mu;
    int count;
    __device__ __forceinline__ void init(double eps0) {  // step_sizes.py:50-57
        log_step = log(eps0); log_bar = log_step; hbar = 0.0; mu = log(10.0 * eps0);
        count = 1;
    }
    __device__ __forceinline__ void update(const RunCfg& P, double accept) {  // step_sizes.py:66-78
        const double w = 1.0 / (count + P.t0);
        hbar = __dadd_rn(__dmul_rn(1.0 - w, hbar), __dmul_rn(w, P.target - accept));
        log_step = mu - __dmul_rn(hbar, sqrt((double)count)) / P.gamma;
        const double mk = pow((double)count, -P.kappa);
        log_bar = __dadd_rn(__dmul_rn(mk, log_step), __dmul_rn(1.0 - mk, log_bar));
        ++count;
    }
    __device__ __forceinline__ double current(bool adapting) const { return exp(adapting ? log_step : log_bar); }  // :60-64
    __device__ __forceinline__ double final_step() const { return exp(log_bar); }
};

// _WeightedVariance.add_sample (quadpotential.py:431-437) of one element, mean part; returns x - old mean
__device__ __forceinline__ double welford_mean(double x, double n, double& mean) {
    const double d0 = x - mean;
    mean = __dadd_rn(mean, d0 / n);
    return d0;
}
__device__ __forceinline__ void welford_add(double x, double n, double& mean, double& m2) {
    const double d0 = welford_mean(x, n, mean);
    m2 = __dadd_rn(m2, __dmul_rn(d0, x - mean));
}

// QuadPotentialDiagAdapt's two estimators (quadpotential.py:335-355): the vector slots of the foreground and background
// (mean, m2) and their weights.  The engines run the element loops; the scalar transitions are here.
struct DiagWindow {
    double fg_n, bg_n;
    int fg_m, fg_v, bg_m, bg_v, k_samples, window;
    // foreground (mean0, var0 * weight) with weight `init_weight`, background empty; slots first .. first + 3
    __device__ __forceinline__ void init(int first, double init_weight, int window_) {
        fg_m = first; fg_v = first + 1; bg_m = first + 2; bg_v = first + 3;
        fg_n = init_weight; bg_n = 0.0;
        k_samples = 0; window = window_;
    }
    // true when the draw is added to both estimators (their weights already counted)
    __device__ __forceinline__ bool add_sample(int discard) {
        if (k_samples <= discard) return false;
        fg_n += 1.0; bg_n += 1.0;
        return true;
    }
    __device__ __forceinline__ bool var_ready() const { return k_samples > window; }
    __device__ __forceinline__ double variance(double m2) const { return fmin(fmax(m2 / fg_n, 1e-12), 1e12); }
    __device__ __forceinline__ bool swap_due() const { return k_samples > 0 && k_samples % window == 0; }
    // the background becomes the foreground; the caller clears the new background's vectors
    __device__ __forceinline__ void swap() {
        const int tm = fg_m, tv = fg_v;
        fg_m = bg_m; fg_v = bg_v; fg_n = bg_n;
        bg_m = tm; bg_v = tv; bg_n = 0.0;
    }
};

// Stats of an iteration that never ran (chain frozen by "Bad initial energy"): zeros / NaN, so caller-provided output
// buffers need no clearing before a run and a reused buffer never shows values of an earlier run.
__device__ __forceinline__ void stats_sentinel(const b200_stats& st, long long o) {
    const double qnan = nan("");
    if (st.depth) st.depth[o] = 0;
    if (st.tree_size) st.tree_size[o] = 0;
    if (st.index_in_trajectory) st.index_in_trajectory[o] = 0;
    if (st.diverging) st.diverging[o] = 0;
    if (st.reached_max_treedepth) st.reached_max_treedepth[o] = 0;
    if (st.step_size) st.step_size[o] = qnan;
    if (st.step_size_bar) st.step_size_bar[o] = qnan;
    if (st.mean_tree_accept) st.mean_tree_accept[o] = qnan;
    if (st.energy) st.energy[o] = qnan;
    if (st.energy_error) st.energy_error[o] = qnan;
    if (st.max_energy_error) st.max_energy_error[o] = qnan;
    if (st.model_logp) st.model_logp[o] = qnan;
}

// The sampler statistics of one draw (nuts.py:478-489, base_hmc.py:275-286)
__device__ __forceinline__ void record_draw_stats(const b200_stats& st, long long o, int depth, int tree_size, int idx,
                                                  bool diverged, bool hit_max, const StepSize& ss, double accept,
                                                  double energy, double energy_error, double max_de, double logp) {
    if (st.depth) st.depth[o] = depth;
    if (st.tree_size) st.tree_size[o] = tree_size;
    if (st.index_in_trajectory) st.index_in_trajectory[o] = idx;
    if (st.diverging) st.diverging[o] = diverged ? 1 : 0;
    if (st.reached_max_treedepth) st.reached_max_treedepth[o] = hit_max ? 1 : 0;
    if (st.step_size) st.step_size[o] = exp(ss.log_step);
    if (st.step_size_bar) st.step_size_bar[o] = exp(ss.log_bar);
    if (st.mean_tree_accept) st.mean_tree_accept[o] = accept;
    if (st.energy) st.energy[o] = energy;
    if (st.energy_error) st.energy_error[o] = energy_error;
    if (st.max_energy_error) st.max_energy_error[o] = max_de;
    if (st.model_logp) st.model_logp[o] = logp;
}

// A frozen chain ("Bad initial energy", base_hmc.py:205-224): the recorded iterations of [t_from, t_to) that never ran are
// NaN draws with sentinel stats.  Output row of iteration t: t - rec_lo.  Team of TS threads.
template <int TS>
__device__ __forceinline__ void freeze_outputs(const RunCfg& P, int chain, int t_from, int t_to, int rec_lo, int T_out,
                                               int lane) {
    for (int t = t_from; t < t_to; ++t) {
        if (!(P.store_warmup || t >= P.tune)) continue;
        const long long o = (long long)chain * T_out + (t - rec_lo);
        for (int i = lane; i < P.n; i += TS) P.draws_out[o * P.n + i] = nan("");
        if (lane == 0) stats_sentinel(P.st, o);
    }
}

// The chain's summary scalars, written once its schedule is over
__device__ __forceinline__ void record_chain_summary(const b200_chain_summary& sm, int chain, long long n_grad, int bad_at,
                                                     const StepSize& ss) {
    if (sm.grad_evals) sm.grad_evals[chain] = n_grad;
    if (sm.bad_energy_at) sm.bad_energy_at[chain] = bad_at;
    if (sm.final_step_size) sm.final_step_size[chain] = ss.final_step();
}

// Standard-normal momentum noise of (chain, iteration `it`, element i): the caller's buffer z, which holds the n_iter
// iterations this call runs, or the counter-based Philox stream.  The lock-step engine always runs whole schedules
// (it0 = 0, n_iter = tune + draws: b200_nuts_run refuses anything else), so both engines index z by `it - it0`.
__device__ __forceinline__ double momentum_z(const RunCfg& P, int chain, int it, int i) {
    return (P.momentum_source == B200_MOMENTUM_HOST_BUFFER)
               ? P.z[((long long)chain * P.n_iter + (it - P.it0)) * P.n + i]
               : philox_normal(P.philox_seed, (uint32_t)(chain + P.chain_offset), (uint32_t)it, (uint32_t)i);
}

// Merge of two multinomial log-weights a (the subtree just built) and b as the lock-step engine carries them:
// logaddexp(a, b) computed through log1p_abs, with d = a - b and e = exp(-|d|), from which the picks take P(a) = w_a / (w_a + w_b)
// (subtree merge) or min(1, w_a / w_b) (top-level pick).
__device__ __forceinline__ double merge_logw(double a, double b, double& d, double& e) {
    d = a - b;
    e = exp(-fabs(d));
    return (d == 0.0) ? a + 0.69314718055994530942 : (isnan(d) ? a + b : fmax(a, b) + log1p_abs(e));
}

}  // namespace b200
