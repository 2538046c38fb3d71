// Generic fused log-density + reverse-mode gradient for a model given as ModelSpec IR (include/b200nuts.h: b200_ir;
// pymc_b200/ir.py).  One device function evaluates ANY model of the closed factor set, so a new model needs no new CUDA;
// it plugs into the same persistent NUTS / leapfrog / logp kernels as the hand-specialised models (same `eval` contract).
//
// It replaces one call of the compiled PyTensor function  q -> (logp, dlogp)  (pymc/model/core.py:232-267) and composes
// the joint density exactly the way the reference does:
//   1. constrain: x = backward(q) per value variable, + log|Jacobian|   (logprob/transforms.py:880-891, :1026-1073)
//   2. logp(x) = sum of factors (model/core.py:688-690), gx = d logp / d x accumulated factor by factor
//   3. chain rule through the transforms: g_q = gx * dx/dq + d log|J| / dq
// Determinism: no atomics.  A likelihood's gradient is PULLED: scalar targets by a team reduction over observations,
// indexed targets (group effects) through a CSR transpose of the index built at model-create time, so every sum has a
// fixed order and results are bit-identical from run to run and independent of how chains are sharded.
//
// Team scratch in global memory (L1/L2 resident), one slice per resident team: x[n] and the per-observation
// d loglik / d eta of the likelihood being processed.
//
// A random dispersion alpha (NegativeBinomial, Gamma) reaches its slot through the same team reduction as a likelihood's
// sigma.  Its normalising terms are not per observation: Gamma's once per evaluation, NegativeBinomial's over a table of
// the distinct nonzero counts (csrc/b200nuts.cu: prepare_ir), with digamma() of common.cuh for the gradient.
#pragma once
#include "../../include/b200nuts.h"
#include "common.cuh"

namespace b200 {

constexpr double kNegBinPoissonAlpha = 1e10;  // above: NegativeBinomial -> Poisson(mu) limit (discrete.py:727-735)

// ---- the likelihood groups prepare_ir and the device branch on, each named after its pymc_b200/ir.py tuple; ranges: static_assert
__host__ __device__ __forceinline__ constexpr bool ir_bounded_liks(int d) { return d == B200_IR_L_CENSORED_NORMAL || d == B200_IR_L_TRUNCATED_NORMAL; }
__host__ __device__ __forceinline__ constexpr bool ir_ordinal_liks(int d) { return d == B200_IR_L_ORDERED_LOGISTIC || d == B200_IR_L_ORDERED_PROBIT; }
static_assert(B200_IR_L_ZERO_INFLATED_POISSON == 12 && B200_IR_L_ZERO_INFLATED_BINOMIAL == 13 && B200_IR_L_ZERO_INFLATED_NEGATIVE_BINOMIAL == 14 &&
              B200_IR_L_HURDLE_POISSON == 15 && B200_IR_L_HURDLE_NEGATIVE_BINOMIAL == 16 && B200_IR_L_HURDLE_GAMMA == 17, "ZI_LIKS, the hurdles last");
__host__ __device__ __forceinline__ constexpr bool ir_zi_liks(int d) { return d >= B200_IR_L_ZERO_INFLATED_POISSON && d <= B200_IR_L_HURDLE_GAMMA; }
__host__ __device__ __forceinline__ constexpr bool ir_hurdle_liks(int d) { return d >= B200_IR_L_HURDLE_POISSON; }  // of a ZI_LIKS id
__host__ __device__ __forceinline__ constexpr int ir_zi_family(int d) {  // ZI_FAMILY: a ZI_LIKS id's family, whose slot (trials, alpha) it takes
    return d == B200_IR_L_ZERO_INFLATED_BINOMIAL ? B200_IR_L_BINOMIAL_LOGIT : d == B200_IR_L_HURDLE_GAMMA ? B200_IR_L_GAMMA_LOG
         : d == B200_IR_L_ZERO_INFLATED_NEGATIVE_BINOMIAL || d == B200_IR_L_HURDLE_NEGATIVE_BINOMIAL ? B200_IR_L_NEGBINOMIAL_LOG : B200_IR_L_POISSON_LOG;
}
__host__ __device__ __forceinline__ constexpr bool ir_weibull_liks(int d) { return d == B200_IR_L_WEIBULL_LOG || d == B200_IR_L_CENSORED_WEIBULL_LOG || d == B200_IR_L_TRUNCATED_WEIBULL_LOG; }
__host__ __device__ __forceinline__ constexpr bool ir_lognormal_liks(int d) { return d == B200_IR_L_LOGNORMAL || d == B200_IR_L_CENSORED_LOGNORMAL || d == B200_IR_L_TRUNCATED_LOGNORMAL; }
static_assert(B200_IR_L_WEIBULL_LOG == 18 && B200_IR_L_LOGNORMAL == 19 && B200_IR_L_CENSORED_WEIBULL_LOG == 20 && B200_IR_L_CENSORED_LOGNORMAL == 21 &&
              B200_IR_L_TRUNCATED_WEIBULL_LOG == 22 && B200_IR_L_TRUNCATED_LOGNORMAL == 23, "SURVIVAL_LIKS");
__host__ __device__ __forceinline__ constexpr bool ir_survival_liks(int d) { return d >= B200_IR_L_WEIBULL_LOG && d <= B200_IR_L_TRUNCATED_LOGNORMAL; }
__host__ __device__ __forceinline__ constexpr bool ir_censored_survival_liks(int d) { return d == B200_IR_L_CENSORED_WEIBULL_LOG || d == B200_IR_L_CENSORED_LOGNORMAL; }
__host__ __device__ __forceinline__ constexpr bool ir_truncated_survival_liks(int d) { return d == B200_IR_L_TRUNCATED_WEIBULL_LOG || d == B200_IR_L_TRUNCATED_LOGNORMAL; }
__host__ __device__ __forceinline__ constexpr bool ir_mixture_liks(int d) { return d == B200_IR_L_NORMAL_MIXTURE || d == B200_IR_L_POISSON_MIXTURE; }
__host__ __device__ __forceinline__ constexpr bool ir_beta_liks(int d) { return d == B200_IR_L_BETA_LOGIT || d == B200_IR_L_BETA_BINOMIAL_LOGIT; }
__host__ __device__ __forceinline__ constexpr bool ir_sigma_liks(int d) { return d == B200_IR_L_NORMAL || d == B200_IR_L_STUDENTT || ir_bounded_liks(d) || d == B200_IR_L_ORDERED_PROBIT || ir_lognormal_liks(d); }
// the likelihoods and transforms that IrModel leaves out and IrExtendedModel evaluates out of line (below)
__host__ __device__ __forceinline__ constexpr bool ir_extended_liks(int d) { return ir_ordinal_liks(d) || ir_zi_liks(d) || ir_mixture_liks(d) || ir_bounded_liks(d) || ir_survival_liks(d) || ir_beta_liks(d); }
static_assert(B200_IR_T_ORDERED == 3 && B200_IR_T_ORDERED_POSITIVE == 4 && B200_IR_T_SIMPLEX == 5, "the last three transforms");
__host__ __device__ __forceinline__ constexpr bool ir_extended_transforms(int t) { return t >= B200_IR_T_ORDERED; }  // ORDERED_TRANSFORMS and simplex

struct IrParamD { int kind, ref; double value; };                     // kind 0: constant; 1: x[ref] (a scalar variable)
struct IrVarD { int offset, size, transform, pad; double lo, hi; };  // pad: a simplex variable's rows (below)
struct IrPriorD { int dist, offset, size, pad; IrParamD p[3]; double c0; };      // c0: per-element constant of the density
                                                                                 // (dirichlet: of the whole vector; pad: the rows)
struct IrFactorD { int offset, size; const int* idx; const int* rowptr; const int* rowobs; };  // CSR: element -> observations
// n_cols > 0: a design term, eta_i += sum_k X[i][k] x[f[0].offset + k], with coef = X row-major [N][n_cols] (the gradient
// reads it) and xt = X column-major [n_cols][N] (the forward pass reads it: consecutive threads take consecutive rows).
struct IrTermD { const double* coef; int n_factors, n_cols; IrFactorD f[3]; const double* xt; };
constexpr int kIrPartDoubles = 256;  // per-team slice partials of a design term's gradient, at the end of the team scratch

// A spectral term (include/b200nuts.h) runs as a design term whose coefficients are b_k = s_k z_k: its device IrTermD has
// n_factors == 3, f[0].offset = the b row and f[1].offset = the g_b row, both in the team slice.  ir_spectral_forward fills
// the b row before any likelihood, so ir_eta and ir_design_row read it as they read a variable; term_grad writes
// g_b = Phi^T r into the g_b row, and ir_spectral_grad takes it back to z, a and l.  One IrSpecD per spectral term, in
// the table in front of the terms (ir_spec_count, ir_specs).
//   log s_k = log a + (log C_D + sum_d log l_d + h(Q_k)) / 2,  Q_k = sum_d l_d^2 omega_kd^2,
//   h = -Q / 2 (EXPQUAD: nu == 0) or -nu log(c + Q) (Matern: nu = (D + 5) / 2, c = 5 or nu = (D + 3) / 2, c = 3),
// so s_k underflows to 0 instead of forming 0 * inf where the density is far below the double range.
struct IrSpecD {
    int z, b_row, gb_row, s_row;  // z's offset in x; the rows b = s z, g_b and s of the team slice
    int M, D, a_ref, ls_ref;      // a_ref: the amplitude's offset in x, or -1 for the constant a
    int ls_size, pad0, pad1, pad2;  // 1 or D: the lengthscale variable at ls_ref; 0: the constants ls[D]
    double a, log_c, nu, c;
    const double* ls;
    const double* omega;  // [M][D]
};
static_assert(sizeof(IrSpecD) % alignof(IrTermD) == 0, "the IrSpecD table sits in front of the terms");
// The terms' allocation is [IrSpecD x n_spec][long long n_spec][IrTermD ...] with IrModel::Params::terms at the first term:
// IrModel and its kernels never look in front of it, so models without spectral terms keep every table and kernel they had.
__host__ __device__ __forceinline__ int ir_spec_count(const IrTermD* terms) { return (int)reinterpret_cast<const long long*>(terms)[-1]; }
__host__ __device__ __forceinline__ const IrSpecD* ir_specs(const IrTermD* terms, int n_spec) {
    return reinterpret_cast<const IrSpecD*>(reinterpret_cast<const long long*>(terms) - 1) - n_spec;
}

// sum_k X[i][k] b[k], k ascending
__device__ __forceinline__ double ir_design_row(const IrTermD& Tm, const double* b, int i, int N) {
    const double* xt = Tm.xt + i;
    double s = 0.0;
    for (int k = 0; k < Tm.n_cols; ++k) s = fma(xt[(long long)k * N], b[k], s);
    return s;
}

// g[k] += sum_i X[i][k] r[i] with the whole team, no atomics.  Columns go TS at a time; a block of kc < TS columns (the last
// one) splits the rows into S = TS / kc interleaved slices, thread t taking column t % kc and rows i = t / kc (mod S), so a
// warp reads adjacent rows of row-major X.  The slice partials meet in `part` and are added in slice order.  Every sum
// has a fixed order, so the result does not depend on the run or on the other teams.
template <int W>
__device__ __forceinline__ void ir_design_grad(const IrTermD& Tm, const double* r, int N, double* g, double* part, int tid) {
    constexpr int TS = 32 * W;
    const int K = Tm.n_cols;
    const double* X = Tm.coef;
    for (int c0 = 0; c0 < K; c0 += TS) {
        const int kc = min(K - c0, TS), S = TS / kc, c = tid % kc, s = tid / kc;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;  // four independent chains, combined in a fixed order
        if (s < S) {
            const double* xc = X + c0 + c;
            int i = s;
            for (; i + 3 * S < N; i += 4 * S) {
                a0 = fma(xc[(long long)i * K], r[i], a0);
                a1 = fma(xc[(long long)(i + S) * K], r[i + S], a1);
                a2 = fma(xc[(long long)(i + 2 * S) * K], r[i + 2 * S], a2);
                a3 = fma(xc[(long long)(i + 3 * S) * K], r[i + 3 * S], a3);
            }
            for (; i < N; i += S) a0 = fma(xc[(long long)i * K], r[i], a0);
        }
        const double a = (a0 + a1) + (a2 + a3);
        if (S == 1) {
            if (s == 0) g[c0 + c] += a;
        } else {  // uniform branch; only the last block can take it
            if (s < S) part[tid] = a;
            team_sync<W>();
            if (tid < kc) {
                double tot = part[c];
                for (int j = 1; j < S; ++j) tot += part[j * kc + c];
                g[c0 + c] += tot;
            }
        }
    }
}
// c0: sum of the constant parts over i.  Random dispersion (sigma_kind REF): Gamma keeps sum_i log y_i in sum_log_y;
// NegativeBinomial keeps the distinct nonzero y values u[k] with their counts cnt[k] (n_tab of them), over which the
// alpha-dependent normalising terms sum_i lgamma(y_i + a) - lgamma(a) and their digamma gradient are evaluated; the
// zero-inflated and hurdle NegativeBinomial use the same table.  hurdle_gamma: sum_log_y = sum of log y_i over y_i > 0
// and n_tab = N+, the number of such y_i.
// Censored Normal: cens[i] = 0 (observed), 1 (y_i at its lower bound), 2 (at its upper bound); the censoring point is y_i
// itself.  Truncated Normal: bnd = [2][N], the lower and upper bound of each observation, -inf / +inf where open.
// Survival likelihoods: y = log y_i; cens as above for the censored forms and null otherwise; bnd of the truncated forms
// holds the bounds themselves (Weibull, 0 / +inf where open) or their logs (LogNormal, -inf / +inf where open).
// Beta: y = the [2][N] block (log y_i, log1p(-y_i)).  BetaBinomial: y = the [2][N] block (y_i, n_i); a random phi keeps the
// distinct nonzero trials in tab_u with their counts in tab_cnt (n_tab of them).
// yoff >= 0: a latent factor (a Normal / StudentT prior whose location is a linear predictor): y_i = x[yoff + i], the
// constrained values of a variable of size N, which also receives d logp / d y_i = -r_i; y is null.  -1: y is data.
struct IrLikD { int dist, n_terms, term0, sigma_kind; long long N; const double* y; const double* sigma_obs; IrParamD sigma;
                double nu, c0, sum_log_y; const double* tab_u; const double* tab_cnt; int n_tab, yoff;
                const signed char* cens; const double* bnd; };
struct IrAr1D { int offset, size; IrParamD phi, sigma; double init_sigma; };

// ---- per-observation pieces, shared by eval's observation loops and the pointwise kernel

// x_f[idx_f[i]]: factor F at observation i (indexed, scalar or elementwise)
__device__ __forceinline__ double ir_factor(const IrFactorD& F, const double* x, int i) {
    return x[F.offset + (F.idx ? F.idx[i] : (F.size == 1 ? 0 : i))];
}

// eta_i = sum_t coef_t[i] prod_f x_f[idx_f[i]] over the block terms[term0 .. term0 + n_terms), t ascending.
// terms is taken by reference so that eval, which passes the member P.terms, loads it inside the loop, after the
// n_terms check, and indexes it with term0 + t; the out-of-line passes pass the block's start with term0 = 0.  Each
// caller thereby keeps the code it had with its own inline loop, and the kernels that reach eval keep their register
// allocation (stack and spills are sensitive to any change in eval's code).
__device__ __forceinline__ double ir_eta(const IrTermD* const& terms, int term0, int n_terms, const double* x, int i,
                                         int N) {
    double eta = 0.0;
    for (int t = 0; t < n_terms; ++t) {
        const IrTermD& Tm = terms[term0 + t];
        if (Tm.n_cols) {
            eta += ir_design_row(Tm, x + Tm.f[0].offset, i, N);
            continue;
        }
        double pr = Tm.coef ? Tm.coef[i] : 1.0;
        for (int f = 0; f < Tm.n_factors; ++f) pr *= ir_factor(Tm.f[f], x, i);
        eta += pr;
    }
    return eta;
}

// x = backward(z) of one element of a log / interval variable, log|dx/dz| added to lj (transforms.py:880-891, :1026-1073)
__device__ __forceinline__ double ir_backward(const IrVarD& V, double z, double& lj) {
    double xv = z;
    if (V.transform == B200_IR_T_LOG) {
        xv = exp(z);
        lj += z;
    } else if (V.transform == B200_IR_T_INTERVAL) {
        xv = V.lo + (V.hi - V.lo) * sigmoid(z);
        lj += log(V.hi - V.lo) - softplus(-z) - softplus(z);
    }
    return xv;
}

// the value of the slot (sigma, the Binomial's trials or alpha) where it is a constant or a scalar variable
__device__ __forceinline__ double ir_slot(const IrLikD& L, const double* x) {
    return (L.sigma_kind == B200_IR_S_REF) ? x[L.sigma.ref] : L.sigma.value;
}

// the scale (or the Binomial's trials) of observation i: its own value, or the slot's sg_s
__device__ __forceinline__ double ir_scale(const IrLikD& L, int i, double sg_s) {
    return (L.sigma_kind == B200_IR_S_OBS) ? L.sigma_obs[i] : sg_s;
}

// The NegativeBinomial (discrete.py:700-745, n = a, p = a / (mu + a)) at d = eta - log a: lse = logaddexp(eta, log a) =
// log a + softplus(d) = eta + softplus(-d), with s = mu / (mu + a) and sc = a / (mu + a) from one exp, so nothing
// overflows for any finite eta.  e = exp(-|d|), l1 = log1p(e), sp = softplus(d) = lse - log a.
struct IrNegBin { double d, e, l1, s, sc, sp; };
__device__ __forceinline__ IrNegBin ir_negbin(double eta, double la) {
    const double d = eta - la, e = exp(-fabs(d)), l1 = log1p(e), h = 1.0 / (1.0 + e);
    return {d, e, l1, d >= 0 ? h : e * h, d >= 0 ? e * h : h, fmax(d, 0.0) + l1};
}

// log p(y_i | eta) of one observation of the eight base families, less the constants of ir_obs_const, added to lp, and
// d / d sigma (NegativeBinomial, Gamma: d / d alpha; the NegativeBinomial's without psi(y + a) - psi(a)) added to s_sig.
// Returns r_i = d / d eta.  It adds in place rather than returning its parts, so eval's running sums take exactly the
// additions written here, in this order, and a family without a sigma adds nothing to s_sig.
__device__ __forceinline__ double ir_base_term(const IrLikD& L, int i, double yi, double eta, double sg_s, double la,
                                               double& lp, double& s_sig) {
    double ri = 0.0;
    switch (L.dist) {
        case B200_IR_L_NORMAL: {  // continuous.py:526-527
            const double sg = ir_scale(L, i, sg_s);
            const double z = (yi - eta) / sg;
            lp += -0.5 * z * z - log(sg);
            ri = z / sg; s_sig += (z * z - 1.0) / sg;
        } break;
        case B200_IR_L_BERNOULLI_LOGIT:  // discrete.py:362-367 in PyTensor's stabilised forms
            lp += yi * eta - softplus(eta);
            ri = yi - sigmoid(eta);
            break;
        case B200_IR_L_POISSON_LOG: {  // discrete.py:581-586
            const double mu = exp(eta);
            lp += yi * eta - mu;
            ri = yi - mu;
        } break;
        case B200_IR_L_STUDENTT: {  // continuous.py:1936-1944
            const double sg = ir_scale(L, i, sg_s);
            const double z = (yi - eta) / sg;
            lp += -log(sg) - 0.5 * (L.nu + 1.0) * log1p(z * z / L.nu);
            ri = (L.nu + 1.0) * z / (sg * (L.nu + z * z)); s_sig += -1.0 / sg + ri * z;
        } break;
        case B200_IR_L_NORMAL_LOGVAR: {  // Normal(0, exp(eta / 2))
            const double w = yi * yi * exp(-eta);
            lp += -0.5 * w - 0.5 * eta;
            ri = 0.5 * w - 0.5;
        } break;
        case B200_IR_L_BINOMIAL_LOGIT: {  // discrete.py:141-152 in PyTensor's stabilised forms
            const double nt = ir_scale(L, i, sg_s);
            lp += yi * eta - nt * softplus(eta);
            ri = yi - nt * sigmoid(eta);
        } break;
        case B200_IR_L_NEGBINOMIAL_LOG:  // the lgamma part is in c0 / eval's alpha terms
            if (sg_s > kNegBinPoissonAlpha) {  // uniform branch: the Poisson(mu) limit
                const double mu = exp(eta);
                lp += yi * eta - mu;
                ri = yi - mu;
            } else {
                const IrNegBin nb = ir_negbin(eta, la);
                lp -= yi * (fmax(-nb.d, 0.0) + nb.l1) + sg_s * nb.sp;
                ri = yi * nb.sc - sg_s * nb.s;                     // a (y - mu) / (mu + a)
                s_sig += 1.0 - nb.sp - nb.sc * (1.0 + yi / sg_s);  // d/da except psi(y + a) - psi(a)
            }
            break;
        case B200_IR_L_GAMMA_LOG: {  // continuous.py:2512-2521, beta = a exp(-eta); the eta-free part: c0 / alpha terms
            const double w = yi * exp(-eta);
            lp -= sg_s * (eta + w);
            ri = sg_s * (w - 1.0);
            s_sig -= eta + w;
        } break;
        default: break;
    }
    return ri;
}

// ---- Beta regression: the rising-factorial sums of a BetaBinomial bracket and of its phi-only part.
// sum_{j<m} log(a + j) and sum_{j<m} 1 / (a + j) of a count m: below kIrBetaSumMax from products P of four factors and
// their a-derivatives D (D / P = the four reciprocals), one log and one division per four terms and no cancellation
// however large a is against m; from m = kIrBetaSumMax on, lgamma(a + m) - lgamma(a) and digamma(a + m) - digamma(a),
// which lose about |lgamma(a)| ulp (DESIGN.md section 6).  P overflows above a ~ 1e76.
constexpr int kIrBetaSumMax = 32;
struct IrRise { double l, d; };
__device__ __forceinline__ IrRise ir_rising(double a, double m) {
    if (m >= kIrBetaSumMax) return {lgamma(a + m) - lgamma(a), digamma(a + m) - digamma(a)};
    const int n = (int)m;
    double l = 0.0, d = 0.0;
    for (int j = 0; j < n; j += 4) {
        double P = 1.0, D = 0.0;
        for (int k = j; k < min(j + 4, n); ++k) {
            const double t = a + k;
            D = fma(D, t, P);
            P *= t;
        }
        l += log(P);
        d += D / P;
    }
    return {l, d};
}

// The per-observation constant of log f(y_i) that eval folds into c0 or the alpha terms (csrc/b200nuts.cu: prepare_ir):
// of a base family, and of the count / positive component f of a zero-inflated or hurdle likelihood at y > 0.
__device__ __forceinline__ double ir_obs_const(const IrLikD& L, int i, double y, double sg_s, double la) {
    switch (L.dist) {
        case B200_IR_L_NORMAL: case B200_IR_L_NORMAL_LOGVAR: return -B200_HALF_LOG_2PI;
        case B200_IR_L_STUDENTT: return lgamma(0.5 * (L.nu + 1.0)) - lgamma(0.5 * L.nu) - 0.5 * log(L.nu * 3.14159265358979323846);
        case B200_IR_L_POISSON_LOG: case B200_IR_L_ZERO_INFLATED_POISSON: case B200_IR_L_HURDLE_POISSON: return -lgamma(y + 1.0);
        case B200_IR_L_BINOMIAL_LOGIT: case B200_IR_L_ZERO_INFLATED_BINOMIAL: {  // binomln(n, y)
            const double nt = ir_scale(L, i, sg_s);
            return lgamma(nt + 1.0) - lgamma(y + 1.0) - lgamma(nt - y + 1.0);
        }
        case B200_IR_L_NEGBINOMIAL_LOG: case B200_IR_L_ZERO_INFLATED_NEGATIVE_BINOMIAL: case B200_IR_L_HURDLE_NEGATIVE_BINOMIAL:
            return sg_s > kNegBinPoissonAlpha ? -lgamma(y + 1.0) : lgamma(y + sg_s) - lgamma(sg_s) - lgamma(y + 1.0);
        case B200_IR_L_GAMMA_LOG: case B200_IR_L_HURDLE_GAMMA: return sg_s * la - lgamma(sg_s) + (sg_s - 1.0) * log(y);
        default: return 0.0;
    }
}

// The per-observation constant of a Beta / BetaBinomial observation that eval folds into c0 or the phi terms, apart from
// ir_obs_const so that IrModel's pointwise kernel keeps its code: lgamma(phi) - log y_i - log1p(-y_i) (L.y holds the two
// logs), or binomln(n, y) + lgamma(phi) - lgamma(n + phi).
__device__ __forceinline__ double ir_beta_const(const IrLikD& L, int i, double phi) {
    const double y = L.y[i], v = L.y[L.N + i];
    if (L.dist == B200_IR_L_BETA_LOGIT) return lgamma(phi) - y - v;
    return lgamma(v + 1.0) - lgamma(y + 1.0) - lgamma(v - y + 1.0) - ir_rising(phi, v).l;
}

// log p(y_i | eta) of one censored / truncated Normal observation without its constant -log(2 pi) / 2 (in c0), with
// r = d / d eta and s = d / d sigma.  Censored (logprob/censoring.py:213-248 over Normal): the Normal density where y_i is
// observed, log Phi(zc) at a bound, zc = z at the lower one and -z at the upper one (normal_lccdf(z) = normal_lcdf(-z)).
// Truncated (continuous.py:720-747): the Normal density minus log(Phi(b) - Phi(a)) of the standardised bounds.  The
// LogNormal likelihoods run the same arithmetic on log y and log bounds (a plain one as censored with no code); their
// -log y_i is in c0.
struct IrBoundedTerm { double lp, r, s; };
__device__ __forceinline__ IrBoundedTerm ir_bounded_term(const IrLikD& L, int i, double eta, double sg) {
    const double z = (L.y[i] - eta) / sg;
    if (L.dist != B200_IR_L_TRUNCATED_NORMAL && L.dist != B200_IR_L_TRUNCATED_LOGNORMAL) {
        const int c = L.cens ? L.cens[i] : 0;
        if (c == 0) return {-0.5 * z * z - log(sg), z / sg, (z * z - 1.0) / sg};
        const double zc = c == 1 ? z : -z;
        const NormalTail t = normal_tail(zc);
        return {t.log_cdf, (c == 1 ? -t.mills : t.mills) / sg, -t.mills * zc / sg};
    }
    const int N = (int)L.N;
    const double a = (L.bnd[i] - eta) / sg, b = (L.bnd[N + i] - eta) / sg;  // an open side stays infinite
    const NormalMass M = normal_log_mass(a, b);
    const double ta = M.ra == 0.0 ? 0.0 : a * M.ra, tb = M.rb == 0.0 ? 0.0 : b * M.rb;  // inf * 0 = 0
    return {-0.5 * z * z - log(sg) - M.log_z, (z + M.rb - M.ra) / sg, (z * z - 1.0 + tb - ta) / sg};
}

// ---- survival observations (continuous.py:2740-2831 / :1461-1480 / :1723-1846).  The Weibull with beta = e^eta, at
// u = log y - eta and t = e^{alpha u} = (y / beta)^alpha:  log f = log alpha - eta + (alpha - 1) u - t,  log S = -t,
// log F = log(1 - e^-t).  log S is written directly (the reference has no Weibull logccdf and takes log(1 - F), which
// loses every digit for small t); log F takes log t - t / 2 where t < 2e-9, so it stays finite after t underflows.  t
// overflowing for y far above beta gives log S = -inf, which is the value.
// log(1 - e^-t) given v = log t and t
__device__ __forceinline__ double ir_log1mexp_neg(double v, double t) {
    return v < -20.0 ? v - 0.5 * t : (t < 0.6931471805599453 ? log(-expm1(-t)) : log1p(-exp(-t)));
}
// t / (e^t - 1) given v = log t and t: 1 as t -> 0, 0 once e^t overflows
__device__ __forceinline__ double ir_t_over_expm1(double v, double t) {
    return v < -20.0 ? 1.0 - 0.5 * t : (v > 700.0 ? 0.0 : t / expm1(t));
}
// One Weibull observation: lp, r = d / d eta and s = d / d alpha.  Uncensored: r = alpha (t - 1), s = 1 / alpha + u - u t;
// right-censored (cens 2): r = alpha t, s = -u t; left-censored (cens 1): r = -alpha t / expm1(t), s = u t / expm1(t).
// Truncated to [A, B]: the density minus log Z, Z = S(A) - S(B) = e^{-tA} (1 - e^{-D}), D = tB - tA taken as
// log D = alpha uB + log(1 - e^{-alpha log(B / A)}) with log(B / A) = log1p((B - A) / A), so a window with D ~ 1e-6 keeps
// its digits; an open side drops its factor (A = 0: log Z = log(1 - e^{-tB}); B = +inf: log Z = -tA).
__device__ __forceinline__ IrBoundedTerm ir_weibull_term(const IrLikD& L, int i, double eta, double a, double la) {
    const double u = L.y[i] - eta, v = a * u, t = exp(v);
    const int c = L.cens ? L.cens[i] : 0;
    if (c == 2) return {-t, a * t, -u * t};
    if (c == 1) {
        const double q = ir_t_over_expm1(v, t);
        return {ir_log1mexp_neg(v, t), -a * q, u * q};
    }
    IrBoundedTerm o{la - eta + (a - 1.0) * u - t, a * (t - 1.0), 1.0 / a + u - u * t};
    if (L.bnd) {  // truncated
        const int N = (int)L.N;
        const double A = L.bnd[i], B = L.bnd[N + i];
        double ta = 0.0, ua = 0.0;
        if (A > 0.0) {  // -log Z gains +tA
            ua = log(A) - eta;
            ta = exp(a * ua);
            o.lp += ta;
            o.r -= a * ta;
            o.s += ua * ta;
        }
        if (B != INFINITY) {  // -log Z gains -log(1 - e^-D)
            const double ub = log(B) - eta, lr = A > 0.0 ? log1p((B - A) / A) : 0.0;
            const double ld = A > 0.0 ? a * ub + log(-expm1(-a * lr)) : a * ub, d = exp(ld);
            const double q = ir_t_over_expm1(ld, d);  // D / expm1(D)
            o.lp -= ir_log1mexp_neg(ld, d);
            o.r += a * q;  // dD / d eta = -alpha D
            o.s -= q * (ub + (A > 0.0 ? lr / expm1(a * lr) : 0.0));  // dD / d alpha = uB tB - uA tA = log(B / A) tA + uB D
        }
    }
    return o;
}

// The observation loop of a censored / truncated Normal or a survival likelihood, out of line: IrExtendedModel::eval calls
// it once per such likelihood, so the erfcx() tail math stays out of eval's own observation loop.  Writes r_i = d logp / d eta_i;
// returns this thread's partial sums of logp and d logp / d sigma.
struct IrPartials { double lp, s_sig; };
template <int W>
__device__ __noinline__ IrPartials ir_bounded_pass(const IrLikD* Lp, const IrTermD* terms, const double* x, double* r,
                                                   double sg_s, int tid) {
    constexpr int TS = 32 * W;
    const IrLikD& L = *Lp;
    const int N = (int)L.N;
    const bool weibull = ir_weibull_liks(L.dist);  // sg_s is alpha
    const double la = weibull ? log(sg_s) : 0.0;
    double lp = 0.0, s_sig = 0.0;
    for (int i = tid; i < N; i += TS) {
        const double eta = ir_eta(terms + L.term0, 0, L.n_terms, x, i, N);
        const IrBoundedTerm b = weibull ? ir_weibull_term(L, i, eta, sg_s, la) : ir_bounded_term(L, i, eta, ir_scale(L, i, sg_s));
        lp += b.lp;
        s_sig += b.s;
        r[i] = b.r;
    }
    return {lp, s_sig};
}

// ---- ordinal observations: OrderedLogistic / OrderedProbit (discrete.py:1231-1432) as the Categorical they build
// (Categorical.logp, :1190-1206).  K = L.nu categories, y_i in 0..K-1; the K-1 cutpoints c are terms[term0 + n_terms]:
// one unindexed factor on a variable of size K-1 (f[0].rowptr / rowobs: the observations of each category, ascending), or
// no factor and coef = the constants.  With a = (c_{y-1} - eta) / s, b = (c_y - eta) / s (c_{-1} = -inf, c_{K-1} = +inf;
// s = 1 for the logistic link), log p = log(F(b) - F(a)):
//   logistic  -softplus(-b) - softplus(a) + log1mexp(a - b), the gap b - a taken from the cutpoints themselves, and the
//             one-sided form at an end category;
//   probit    normal_log_mass(a, b).
// The reference forms p in probability space (compute_p, :1312-1326 / :1416-1432) and takes its log, so it returns -inf
// where F(b) - F(a) underflows or cancels; this stays finite for every finite eta.
// Returns lp, rs = s d lp / d eta, w = d lp / d c_y (so d lp / d c_{y-1} = -rs / s - w) and ds = d lp / d s.
struct IrOrdinalTerm { double lp, rs, w, ds; };
__device__ __forceinline__ IrOrdinalTerm ir_ordinal_term(const IrLikD& L, const IrTermD& C, const double* x, int i, double eta,
                                                         double s) {
    const int K = (int)L.nu, y = (int)L.y[i];
    const double* c = C.n_factors ? x + C.f[0].offset : C.coef;
    const bool lo_open = y == 0, hi_open = y == K - 1;
    const double a = lo_open ? -INFINITY : (c[y - 1] - eta) / s, b = hi_open ? INFINITY : (c[y] - eta) / s;
    if (L.dist == B200_IR_L_ORDERED_PROBIT) {
        const NormalMass M = normal_log_mass(a, b);
        const double ta = M.ra == 0.0 ? 0.0 : a * M.ra, tb = M.rb == 0.0 ? 0.0 : b * M.rb;  // inf * 0 = 0
        return {M.log_z, M.ra - M.rb, M.rb / s, (ta - tb) / s};
    }
    const double sa = lo_open ? 0.0 : sigmoid(a), sb = hi_open ? 0.0 : sigmoid(-b);  // F(a), 1 - F(b)
    double lp = (lo_open ? 0.0 : -softplus(a)) + (hi_open ? 0.0 : -softplus(-b)), w = sb;
    if (!lo_open && !hi_open) {
        const double gap = (c[y] - c[y - 1]) / s;  // b - a without the cancellation of forming it from a and b
        lp += log(-expm1(-gap));
        w += 1.0 / expm1(gap);
    }
    return {lp, sa - sb, w, 0.0};
}

// The observation loop of an ordinal likelihood, out of line like ir_bounded_pass.  Writes r_i = d logp / d eta_i and
// w_i = d logp / d c_{y_i}; returns this thread's partial sums of logp and d logp / d sigma.
template <int W>
__device__ __noinline__ IrPartials ir_ordinal_pass(const IrLikD* Lp, const IrTermD* terms, const double* x, double* r,
                                                   double* w, double sg_s, int tid) {
    constexpr int TS = 32 * W;
    const IrLikD& L = *Lp;
    const int N = (int)L.N;
    const IrTermD& C = terms[L.term0 + L.n_terms];
    double lp = 0.0, s_sig = 0.0;
    for (int i = tid; i < N; i += TS) {
        const double eta = ir_eta(terms + L.term0, 0, L.n_terms, x, i, N);
        const double s = ir_scale(L, i, L.sigma_kind == B200_IR_S_NONE ? 1.0 : sg_s);  // the logistic link: s = 1
        const IrOrdinalTerm o = ir_ordinal_term(L, C, x, i, eta, s);
        lp += o.lp;
        s_sig += o.ds;
        r[i] = o.rs / s;
        w[i] = o.w;
    }
    return {lp, s_sig};
}

// d logp / d c_k = sum of w_i over category k + sum of (-r_i - w_i) over category k + 1, each over the category's
// observations in ascending order (the CSR of the cutpoint term), one thread per cutpoint: no atomics, a fixed order.
template <int W>
__device__ __noinline__ void ir_cutpoint_grad(const IrLikD* Lp, const IrTermD* terms, const double* r, const double* w,
                                              double* g, int tid) {
    constexpr int TS = 32 * W;
    const IrLikD& L = *Lp;
    const IrFactorD& F = terms[L.term0 + L.n_terms].f[0];
    for (int k = tid; k < F.size; k += TS) {
        double a = 0.0;
        for (int e = F.rowptr[k]; e < F.rowptr[k + 1]; ++e) a += w[F.rowobs[e]];
        for (int e = F.rowptr[k + 1]; e < F.rowptr[k + 2]; ++e) {
            const int i = F.rowobs[e];
            a -= r[i] + w[i];
        }
        g[F.offset + k] += a;
    }
}

// ---- zero-inflated and hurdle observations (mixture.py:560-1035).  psi is the probability of the count / positive
// component f, the family at mu = exp(eta) (Binomial: p = sigmoid(eta)), P0 = f(0):
//   zero-inflated (mixture_logprob, :469-494)  y = 0: logaddexp(log(1 - psi), log psi + log P0);  y > 0: log psi + log f(y)
//   hurdle (marginal_hurdle_logprob, :846-870) y = 0: log(1 - psi);  y > 0: log psi + log f(y) - log(1 - P0), the discrete
//                                              component being Truncated(f, lower=1) (:826-829); Gamma has P0 = 0
// log P0 is -e^eta (Poisson), -n softplus(eta) (Binomial), -a softplus(eta - log a) (NegativeBinomial, whose a > 1e10
// Poisson limit is kept).  log(1 - P0) = log1mexp(log P0), and log m (m = -log P0) where m is below 1e-304, so the density
// stays finite for every finite eta.  The constants of f (-lgamma(y + 1), binomln(n, y), and the NegativeBinomial's
// lgamma(y + a) - lgamma(a), the Gamma normaliser over the y > 0) are in c0 / the alpha terms of eval, and in
// ir_obs_const.  Returns lp, r = d lp / d eta, dz = d lp / d zeta, dpsi = d lp / d psi, da = d lp / d alpha.
//
// psi, log psi and log(1 - psi) at observation i from the psi block pt = terms + term0 + n_terms: m = nu = 0, psi itself,
// one constant (coef[0]) or one scalar variable; m >= 1, psi = sigmoid(zeta), zeta the sum of the m terms, with log psi =
// -softplus(-zeta) and log(1 - psi) = -softplus(zeta).
struct IrPsi { double psi, lpsi, l1psi; };
__device__ __forceinline__ IrPsi ir_psi(const IrTermD* pt, int m, const double* x, int i, int N) {
    if (m == 0) {
        const double psi = pt->n_factors ? x[pt->f[0].offset] : pt->coef[0];
        return {psi, log(psi), log1p(-psi)};
    }
    const double z = ir_eta(pt, 0, m, x, i, N);
    return {sigmoid(z), -softplus(-z), -softplus(z)};
}
struct IrZiTerm { double lp, r, dz, dpsi, da; };
__device__ __forceinline__ IrZiTerm ir_zi_term(int dist, double y, double eta, double nt, double a, double la, const IrPsi& ps) {
    const double psi = ps.psi, lpsi = ps.lpsi, l1psi = ps.l1psi;
    // the family: lf = log f(y) less its constants, rf / af = its eta / alpha derivatives; lP0 = log P0 with r0 / a0;
    // lm = log(-lP0)
    double lf, rf, af = 0.0, lP0 = -INFINITY, r0 = 0.0, a0 = 0.0, lm = INFINITY;
    if (dist == B200_IR_L_HURDLE_GAMMA) {  // continuous.py:2512-2521, beta = a exp(-eta)
        const double w = y * exp(-eta);
        lf = -a * (eta + w);
        rf = a * (w - 1.0);
        af = -(eta + w);
    } else if (dist == B200_IR_L_ZERO_INFLATED_BINOMIAL) {  // discrete.py:141-152 in PyTensor's stabilised forms
        lP0 = -nt * softplus(eta);
        r0 = -nt * sigmoid(eta);
        lf = y * eta + lP0;
        rf = y + r0;
    } else if (dist != B200_IR_L_ZERO_INFLATED_POISSON && dist != B200_IR_L_HURDLE_POISSON && a <= kNegBinPoissonAlpha) {  // discrete.py:700-745
        const IrNegBin nb = ir_negbin(eta, la);
        lP0 = -a * nb.sp;
        r0 = -a * nb.s;
        a0 = nb.s - nb.sp;
        lf = lP0 - y * (fmax(-nb.d, 0.0) + nb.l1);
        rf = y * nb.sc + r0;
        af = 1.0 - nb.sp - nb.sc * (1.0 + y / a);
        lm = la + (nb.d < -30.0 ? nb.d - 0.5 * nb.e : log(nb.sp));  // log softplus(d) = d - e^d / 2 to rounding below -30
    } else {  // discrete.py:581-586, and the NegativeBinomial's Poisson limit (:727-735)
        const double mu = exp(eta);
        lP0 = -mu;
        r0 = -mu;
        lf = y * eta - mu;
        rf = y - mu;
        lm = eta;
    }
    const bool hurdle = ir_hurdle_liks(dist);
    if (y == 0.0) {
        if (hurdle) return {l1psi, 0.0, -psi, -exp(-l1psi), 0.0};
        const double t = lpsi + lP0, u = t - l1psi;  // u: the log-odds of the count component at a zero
        const double lp = fmax(t, l1psi) + log1p(exp(-fabs(u)));
        const double w = sigmoid(u);
        // d/dpsi = -(1 - P0) / ((1 - psi) + psi P0): one quotient, finite as psi -> 1
        return {lp, w * r0, w - psi, expm1(lP0) * exp(-lp), w * a0};
    }
    IrZiTerm o{lpsi + lf, rf, 1.0 - psi, exp(-lpsi), af};
    if (hurdle && dist != B200_IR_L_HURDLE_GAMMA) {  // - log(1 - P0)
        if (lm < -700.0) {  // m = -log P0 < 1e-304: log(1 - e^-m) = log m, d log m / d eta = 1, d log m / d a = 0
            o.lp -= lm;
            o.r -= 1.0;
        } else {
            const double q = 1.0 / expm1(-lP0);
            o.lp -= lP0 > -0.6931471805599453 ? log(-expm1(lP0)) : log1p(-exp(lP0));
            o.r += r0 * q;
            o.da += a0 * q;
        }
    }
    return o;
}

// The observation loop of a zero-inflated / hurdle likelihood, out of line like ir_bounded_pass.  Writes r_i = d logp /
// d eta_i and, for a logit psi, z_i = d logp / d zeta_i; returns this thread's partial sums of logp, d logp / d alpha and
// d logp / d psi.
struct IrZiPartials { double lp, s_a, s_psi; };
template <int W>
__device__ __noinline__ IrZiPartials ir_zi_pass(const IrLikD* Lp, const IrTermD* terms, const double* x, double* r,
                                                double* zr, double sg_s, double la, int tid) {
    constexpr int TS = 32 * W;
    const IrLikD& L = *Lp;
    const int N = (int)L.N, m = (int)L.nu;
    const IrTermD* pt = terms + L.term0 + L.n_terms;  // the psi block
    IrPsi ps{0.0, 0.0, 0.0};
    if (m == 0) ps = ir_psi(pt, 0, x, 0, N);
    double lp = 0.0, s_a = 0.0, s_psi = 0.0;
    for (int i = tid; i < N; i += TS) {
        const double eta = ir_eta(terms + L.term0, 0, L.n_terms, x, i, N);
        if (m > 0) ps = ir_psi(pt, m, x, i, N);
        const double nt = ir_scale(L, i, sg_s);
        const IrZiTerm o = ir_zi_term(L.dist, L.y[i], eta, nt, sg_s, la, ps);
        lp += o.lp;
        s_a += o.da;
        s_psi += o.dpsi;
        r[i] = o.r;
        if (m > 0) zr[i] = o.dz;
    }
    return {lp, s_a, s_psi};
}

// ---- the ordered transform (transforms.py:79-120): x_0 = z_0 (positive: e^{z_0}), x_k = x_{k-1} + e^{z_k}; log|J| =
// sum_{k>=1} z_k (positive: sum_k z_k).  Not elementwise, so one thread of the team runs it, k ascending (np.cumsum's
// order): O(size) serial work per evaluation, for vectors as short as cutpoints are.
__device__ __noinline__ double ir_ordered_forward(const IrVarD* Vp, const double* q, double* x) {
    const int o = Vp->offset, n = Vp->size;
    const bool pos = Vp->transform == B200_IR_T_ORDERED_POSITIVE;
    double acc = pos ? exp(q[o]) : q[o], lj = pos ? q[o] : 0.0;
    x[o] = acc;
    for (int k = 1; k < n; ++k) {
        const double z = q[o + k];
        acc += exp(z);
        lj += z;
        x[o + k] = acc;
    }
    return lj;
}

// The chain rule through it, in place on g: d/dz_j = e^{z_j} sum_{k>=j} g_k + 1 for j >= 1 (and j = 0 when positive), and
// d/dz_0 = sum_k g_k otherwise.  The reverse cumulative sum runs k descending, on one thread.
__device__ __noinline__ void ir_ordered_chain(const IrVarD* Vp, const double* q, double* g) {
    const int o = Vp->offset, n = Vp->size;
    const bool pos = Vp->transform == B200_IR_T_ORDERED_POSITIVE;
    double s = 0.0;
    for (int k = n - 1; k >= 0; --k) {
        s += g[o + k];
        g[o + k] = (k == 0 && !pos) ? s : fma(exp(q[o + k]), s, 1.0);
    }
}

// ---- the simplex transform (transforms.py:1091-1116): a variable of size K - 1, w = softmax([z, -sum z]).  Its K weights
// never live at the variable's offset of x: V.pad is the offset in the team slice of two rows of K, lw = log w_k and
// G = d logp / d log w_k, which the Dirichlet prior and the mixture passes read and add to.  The forward pass forms
// log w_k = z_k - lse(z), finite where w_k underflows; log|J| = log K + sum_k log w_k (the reference's log_jac_det), whose
// d / d log w_k = 1 starts G.  One thread, k ascending, like the ordered transform.
__device__ __noinline__ double ir_simplex_forward(const IrVarD* Vp, const double* q, double* x) {
    const int o = Vp->offset, K = Vp->size + 1;
    double* lw = x + Vp->pad;
    double* G = lw + K;
    double zs = 0.0, m = -INFINITY;
    for (int k = 0; k < K - 1; ++k) {
        zs += q[o + k];
        m = fmax(m, q[o + k]);
    }
    m = fmax(m, -zs);
    double s = 0.0;
    for (int k = 0; k < K; ++k) s += exp((k < K - 1 ? q[o + k] : -zs) - m);
    const double lse = m + log(s);
    double lj = log((double)K);
    for (int k = 0; k < K; ++k) {
        lw[k] = (k < K - 1 ? q[o + k] : -zs) - lse;
        lj += lw[k];
        G[k] = 1.0;
    }
    return lj;
}

// The Dirichlet prior of a simplex variable (multivariate.py:557-585): c0 + (a - 1) sum_k log w_k, with d / d log w_k = a - 1
// added to G.  One thread, k ascending.
__device__ __noinline__ double ir_dirichlet(const IrPriorD* Fp, double* x) {
    const int K = Fp->size + 1;
    const double am1 = Fp->p[0].value - 1.0;
    double* lw = x + Fp->pad;
    double s = 0.0;
    for (int j = 0; j < K; ++j) {
        s += lw[j];
        lw[K + j] += am1;
    }
    return fma(am1, s, Fp->c0);
}

// The chain rule through it: d/dz_j = (G_j - w_j S) - (G_K - w_K S), S = sum_k G_k, with no division by any w.
__device__ __noinline__ void ir_simplex_chain(const IrVarD* Vp, const double* x, double* g) {
    const int o = Vp->offset, K = Vp->size + 1;
    const double* lw = x + Vp->pad;
    const double* G = lw + K;
    double S = 0.0;
    for (int k = 0; k < K; ++k) S += G[k];
    const double last = G[K - 1] - exp(lw[K - 1]) * S;
    for (int j = 0; j < K - 1; ++j) g[o + j] = (G[j] - exp(lw[j]) * S) - last;
}

// The InverseGamma prior (continuous.py:2631-2640): c0 - (alpha + 1) log x - beta / x per element, c0 = alpha log beta -
// lgamma(alpha), with d / dx = -(alpha + 1) / x + beta / x^2.  Team-strided over the elements; returns this thread's part.
__device__ __noinline__ double ir_inversegamma(const IrPriorD* Fp, const double* x, double* g, int tid, int TS) {
    const int o = Fp->offset, n = Fp->size;
    const double a1 = Fp->p[0].value + 1.0, b = Fp->p[1].value, c0 = Fp->c0;
    double lp = 0.0;
    for (int j = tid; j < n; j += TS) {
        const double xv = x[o + j], ix = 1.0 / xv;
        lp += c0 - a1 * log(xv) - b * ix;
        g[o + j] += ix * (b * ix - a1);
    }
    return lp;
}

// h'(Q) of a spectral term's log density (see IrSpecD)
__device__ __forceinline__ double ir_spectral_dh(const IrSpecD& S, double Q) { return S.nu == 0.0 ? -0.5 : -S.nu / (S.c + Q); }

// Q_k = sum_d (l_d omega_kd)^2, d ascending
__device__ __forceinline__ double ir_spectral_q(const IrSpecD& S, const double* ls, int ls_step, int k) {
    double Q = 0.0;
    for (int d = 0; d < S.D; ++d) {
        const double t = ls[d * ls_step] * S.omega[(long long)k * S.D + d];
        Q = fma(t, t, Q);
    }
    return Q;
}

// the lengthscales of S as this evaluation sees them, with the step between them (0: one isotropic variable)
__device__ __forceinline__ const double* ir_spectral_ls(const IrSpecD& S, const double* x, int& step) {
    step = S.ls_size == 1 ? 0 : 1;
    return S.ls_size ? x + S.ls_ref : S.ls;
}

// Every spectral term's rows for this evaluation: s_k, b_k = s_k z_k, and g_b_k = 0.  Team-strided over k; the caller
// synchronises the team before the rows are read.
__device__ __noinline__ void ir_spectral_forward(const IrSpecD* Sp, int n_spec, double* x, int tid, int TS) {
    for (int j = 0; j < n_spec; ++j) {
        const IrSpecD& S = Sp[j];
        int step;
        const double* ls = ir_spectral_ls(S, x, step);
        double base = S.log_c;
        for (int d = 0; d < S.D; ++d) base += log(ls[d * step]);
        base = fma(0.5, base, log(S.a_ref >= 0 ? x[S.a_ref] : S.a));
        for (int k = tid; k < S.M; k += TS) {
            const double Q = ir_spectral_q(S, ls, step, k);
            const double h = S.nu == 0.0 ? -0.5 * Q : -S.nu * log(S.c + Q);
            const double sk = exp(fma(0.5, h, base));
            x[S.s_row + k] = sk;
            x[S.b_row + k] = sk * x[S.z + k];
            x[S.gb_row + k] = 0.0;
        }
    }
}

// The chain rule from g_b (complete in the g_b rows) to z, a and l: with w_k = z_k s_k g_b_k,
//   d/dz_k = s_k g_b_k,  d/da = sum_k w_k / a,  d/dl_d = sum_k w_k / (2 l_d) + l_d sum_k w_k omega_kd^2 h'(Q_k)
// (an isotropic l takes the sum over d).  Each sum is a team reduction in a fixed order; a k whose s_k underflowed adds
// nothing.
template <int W>
__device__ __noinline__ void ir_spectral_grad(const IrSpecD* Sp, int n_spec, const double* x, double* g, int tid, double* red) {
    constexpr int TS = 32 * W;
    for (int j = 0; j < n_spec; ++j) {
        const IrSpecD& S = Sp[j];
        double sw = 0.0;
        for (int k = tid; k < S.M; k += TS) {
            const double sg = x[S.s_row + k] * x[S.gb_row + k];
            g[S.z + k] += sg;
            sw = fma(x[S.z + k], sg, sw);
        }
        if (S.a_ref < 0 && S.ls_size == 0) continue;  // uniform branch: constant hyperparameters
        const double tw = team_sum<W>(sw, tid, red);
        if (tid == 0 && S.a_ref >= 0) g[S.a_ref] += tw / x[S.a_ref];
        if (S.ls_size == 0) continue;
        int step;
        const double* ls = ir_spectral_ls(S, x, step);
        for (int d = 0; d < S.D; ++d) {
            double sd = 0.0;
            for (int k = tid; k < S.M; k += TS) {
                const double w = x[S.z + k] * x[S.s_row + k] * x[S.gb_row + k];
                if (w == 0.0) continue;
                const double om = S.omega[(long long)k * S.D + d];
                sd = fma(w * om * om, ir_spectral_dh(S, ir_spectral_q(S, ls, step, k)), sd);
            }
            const double td = team_sum<W>(sd, tid, red);
            const double l = ls[d * step];
            if (tid == 0) g[S.ls_ref + d * step] += fma(l, td, tw / (2.0 * l));
        }
    }
}

// ---- finite mixtures (mixture.py:469-494): log p(y_i) = lse_k(l_ik), l_ik = log w_k + log f_k(y_i), over K = L.nu
// components, with the weights, component and (Normal) sigma blocks at terms[term0 + n_terms ..] (include/b200nuts.h).
// f_k is Normal(eta + mu_k, sigma_k) or Poisson(lam_k e^eta), less the constants -log(2 pi) / 2 and -lgamma(y + 1) (in c0:
// they leave the lse unchanged).  The block pointers: lw (x + the simplex row, or the host-logged constants), G (null for
// constant weights), the components c and sigma s with their gradient targets (null for constants).
struct IrMix { const double* lw; double* G; const double* c; double* gc; const double* s; double* gs; bool s_vec; };
__device__ __forceinline__ IrMix ir_mix_block(const IrLikD& L, const IrTermD* terms, const double* x, double* g) {
    const IrTermD* b = terms + L.term0 + L.n_terms;
    const int K = (int)L.nu;
    IrMix M{b[0].n_factors ? x + b[0].f[0].offset : b[0].coef, b[0].n_factors ? (double*)x + b[0].f[0].offset + K : nullptr,
            b[1].n_factors ? x + b[1].f[0].offset : b[1].coef, b[1].n_factors && g ? g + b[1].f[0].offset : nullptr,
            nullptr, nullptr, true};
    if (L.dist == B200_IR_L_NORMAL_MIXTURE) {
        M.s = b[2].n_factors ? x + b[2].f[0].offset : b[2].coef;
        M.gs = b[2].n_factors && g ? g + b[2].f[0].offset : nullptr;
        M.s_vec = !b[2].n_factors || b[2].f[0].size > 1;
    }
    return M;
}
// log f_k(y) less its constant, with d / d eta (= d / d mu_k for the Normal), d / d lam_k or d / d sigma_k in dt.
struct IrMixTerm { double lf, de, dc, ds; };
__device__ __forceinline__ IrMixTerm ir_mix_term(int dist, const IrMix& M, int k, double y, double eta) {
    if (dist == B200_IR_L_NORMAL_MIXTURE) {
        const double sg = M.s[M.s_vec ? k : 0], z = (y - eta - M.c[k]) / sg;
        return {-0.5 * z * z - log(sg), z / sg, z / sg, (z * z - 1.0) / sg};
    }
    const double lam = M.c[k], mu = lam * exp(eta);
    return {y * (log(lam) + eta) - mu, y - mu, (y - mu) / lam, 0.0};
}
// lse_i and r_i = sum_k rho_ik d log f_k / d eta with the max-shifted sum formed in one pass over k (the running maximum
// rescales the partial sums); a term l = -inf (a component of weight 0, or a density that underflows to 0) is skipped, so
// it adds nothing and no NaN, as logsumexp does.
struct IrMixObs { double lse, r; };
__device__ __forceinline__ IrMixObs ir_mix_obs(int dist, int K, const IrMix& M, double y, double eta) {
    double m = -INFINITY, s = 0.0, rr = 0.0;
    for (int k = 0; k < K; ++k) {
        if (M.lw[k] == -INFINITY) continue;
        const IrMixTerm t = ir_mix_term(dist, M, k, y, eta);
        const double l = M.lw[k] + t.lf;
        if (l == -INFINITY) continue;
        if (l > m) {
            const double c = exp(m - l);
            s = fma(s, c, 1.0);
            rr = fma(rr, c, t.de);
            m = l;
        } else {
            const double e = exp(l - m);
            s += e;
            rr = fma(e, t.de, rr);
        }
    }
    return {m + log(s), rr / s};
}

// The observation loop of a mixture, out of line like ir_zi_pass: r_i = d logp / d eta_i, lse_i and eta_i (in the rows
// lr = [lse | eta], 2N doubles), then one team reduction per component k, ascending, that recomputes l_ik from the stored
// eta_i and lse_i and pulls sum_i rho_ik into G_k, sum_i rho_ik
// d log f_k / d theta_k into the component and sum_i rho_ik d log f_k / d sigma_k into sigma: a fixed order, no atomics,
// no bound on K.  Returns this thread's partial sum of logp.
template <int W>
__device__ __noinline__ double ir_mixture_pass(const IrLikD* Lp, const IrTermD* terms, const double* x, double* r, double* lr,
                                               double* g, int tid, double* red) {
    constexpr int TS = 32 * W;
    const IrLikD& L = *Lp;
    const int N = (int)L.N, K = (int)L.nu;
    const IrMix M = ir_mix_block(L, terms, x, g);
    double* er = lr + N;
    double lp = 0.0;
    for (int i = tid; i < N; i += TS) {
        const double eta = ir_eta(terms + L.term0, 0, L.n_terms, x, i, N);
        const IrMixObs o = ir_mix_obs(L.dist, K, M, L.y[i], eta);
        lp += o.lse;
        r[i] = o.r;
        lr[i] = o.lse;
        er[i] = eta;
    }
    team_sync<W>();
    for (int k = 0; k < K; ++k) {
        if (M.lw[k] == -INFINITY) continue;  // uniform: a dropped component
        double a[3] = {0.0, 0.0, 0.0};
        for (int i = tid; i < N; i += TS) {  // each thread reads back the rows it wrote
            const IrMixTerm t = ir_mix_term(L.dist, M, k, L.y[i], er[i]);
            const double l = M.lw[k] + t.lf;
            if (l == -INFINITY) continue;  // rho = 0, and its derivatives may be infinite
            const double rho = exp(l - lr[i]);
            a[0] += rho;
            a[1] = fma(rho, t.dc, a[1]);
            a[2] = fma(rho, t.ds, a[2]);
        }
        team_sum_n<W>(a, tid, red);
        if (tid == 0) {
            if (M.G) M.G[k] += a[0];
            if (M.gc) M.gc[k] += a[1];
            if (M.gs) M.gs[M.s_vec ? k : 0] += a[2];
        }
        team_sync<W>();
    }
    return lp;
}

// ---- Beta regression (continuous.py:1131-1262 at alpha = mu nu, beta = (1 - mu) nu, :1238-1240; discrete.py:178-262):
// mu = sigmoid(eta), a = phi mu and b = phi (1 - mu) = phi sigmoid(-eta), both from one e = exp(-|eta|) so that 1 - mu
// never cancels, and mu (1 - mu) = e / (1 + e)^2.  The brackets of a BetaBinomial are ir_rising (above).
// One observation: lp, r = d / d eta and s = d / d phi, less the parts that are not per observation.
//   beta_logit           (a - 1) log y + (b - 1) log1p(-y) - lgamma(a) - lgamma(b) without -log y - log1p(-y) (c0) and
//                        lgamma(phi) (c0, or once per evaluation), s without psi(phi).  L.y is the [2][N] block
//                        (log y, log1p(-y)), formed on the host.
//   beta_binomial_logit  [lgamma(y + a) - lgamma(a)] + [lgamma(n - y + b) - lgamma(b)] without binomln(n, y) (c0) and
//                        lgamma(phi) - lgamma(n + phi) (c0, or over the distinct-trials table), s without psi(phi) -
//                        psi(n + phi).  L.y is the [2][N] block (y, trials); a bracket is 0 at y = 0 / y = n (m = 0).
__device__ __forceinline__ IrBoundedTerm ir_beta_term(const IrLikD& L, int i, double eta, double phi) {
    const int N = (int)L.N;
    const double e = exp(-fabs(eta)), h = 1.0 / (1.0 + e);
    const double mu = eta >= 0 ? h : e * h, mc = eta >= 0 ? e * h : h;  // sigmoid(eta), sigmoid(-eta)
    const double a = phi * mu, b = phi * mc, w = phi * (e * h * h);      // w = phi mu (1 - mu) = da / d eta = -db / d eta
    if (L.dist == B200_IR_L_BETA_LOGIT) {
        const double ly = L.y[i], l1y = L.y[N + i];
        const double ua = ly - digamma(a), ub = l1y - digamma(b);
        return {a * ly + b * l1y - lgamma(a) - lgamma(b), w * (ua - ub), mu * ua + mc * ub};
    }
    const double y = L.y[i], n = L.y[N + i];
    const IrRise A = ir_rising(a, y), B = ir_rising(b, n - y);
    return {A.l + B.l, w * (A.d - B.d), mu * A.d + mc * B.d};
}

// The observation loop of a Beta / BetaBinomial likelihood, out of line like ir_bounded_pass, with the phi-only terms of a
// random phi: N lgamma(phi) and N psi(phi) once (Beta), or -sum_{j<u} log(phi + j) and its derivative over the distinct
// nonzero trials u with their counts (BetaBinomial), team-strided in a fixed order.  Writes r_i = d logp / d eta_i;
// returns this thread's partial sums of logp and d logp / d phi.
template <int W>
__device__ __noinline__ IrPartials ir_beta_pass(const IrLikD* Lp, const IrTermD* terms, const double* x, double* r,
                                                double phi, int tid) {
    constexpr int TS = 32 * W;
    const IrLikD& L = *Lp;
    const int N = (int)L.N;
    double lp = 0.0, s = 0.0;
    for (int i = tid; i < N; i += TS) {
        const double eta = ir_eta(terms + L.term0, 0, L.n_terms, x, i, N);
        const IrBoundedTerm b = ir_beta_term(L, i, eta, phi);
        lp += b.lp;
        s += b.s;
        r[i] = b.r;
    }
    if (L.sigma_kind == B200_IR_S_REF) {  // uniform branch
        if (L.dist == B200_IR_L_BETA_LOGIT) {
            if (tid == 0) {
                lp = fma((double)N, lgamma(phi), lp);
                s = fma((double)N, digamma(phi), s);
            }
        } else {
            for (int k = tid; k < L.n_tab; k += TS) {
                const double c = L.tab_cnt[k];
                const IrRise R = ir_rising(phi, L.tab_u[k]);
                lp = fma(-c, R.l, lp);
                s = fma(-c, R.d, s);
            }
        }
    }
    return {lp, s};
}

// IrModel evaluates every factor of the closed set except the likelihoods of ir_extended_liks and the transforms of
// ir_extended_transforms; IrExtendedModel (below) is the same function with those added, each out of line.  A kernel's
// register allocation covers every function it can reach, and the tail math takes about 128 registers, so the engine
// instantiates its kernels twice and runs a model on IrExtendedModel only when it has one of them (b200_model.ir_extended):
// every other IR model keeps the kernels it had before.
struct IrModel {
    static constexpr bool kEvalOutOfLine = true;  // eval is __noinline__ (see nuts_model_eval)
    struct Params {
        const IrVarD* vars; const IrPriorD* priors; const IrLikD* liks; const IrTermD* terms; const IrAr1D* ar1;
        int n_vars, n_priors, n_liks, n_ar1, n;
        double* scratch;            // [slots][stride]
        long long stride;           // doubles per team: n_pad + max N (+ max N of the ordinal and logit-psi likelihoods)
                                    // (+ kIrPartDoubles with a design term)
        int n_pad;
        int ord_row;                // offset of the second per-observation row in the team slice (0: none): an ordinal
                                    // likelihood's w, or the d logp / d zeta of a logit psi; likelihoods take turns
    };
    __host__ __device__ static size_t shared_bytes(const Params&) { return 0; }
    __device__ static void stage(const Params&, char*, uint64_t*) {}

    __device__ static __forceinline__ double par(const IrParamD& p, const double* x) { return p.kind ? x[p.ref] : p.value; }

    // The gradient of every (term, factor) of the block terms[term0 .. term0 + n_terms) of length N, given r_i = d logp /
    // d (the block's sum)_i: d sum_i / d x_f = coef * (other factors).  A likelihood's predictor runs it with its r row,
    // the logit of a zero-inflated / hurdle psi with its zeta row.  The caller has synchronised the team after writing r.
    template <int W, bool EXTENDED = false>
    __device__ __forceinline__ static void term_grad(const Params& P, int term0, int n_terms, const double* r, int N,
                                                     double* x, double* g_s, int tid, double* red) {
        constexpr int TS = 32 * W;
        for (int t = 0; t < n_terms; ++t) {
            const IrTermD& Tm = P.terms[term0 + t];
            if (Tm.n_cols) {  // uniform branch: the residuals r are complete after the caller's barrier
                double* gt = g_s + Tm.f[0].offset;
                if constexpr (EXTENDED) {
                    if (Tm.n_factors == 3) gt = x + Tm.f[1].offset;  // a spectral term: Phi^T r into its g_b row
                }
                ir_design_grad<W>(Tm, r, N, gt, x + P.stride - kIrPartDoubles, tid);
                team_sync<W>();
                continue;
            }
            for (int f = 0; f < Tm.n_factors; ++f) {
                const IrFactorD& Fc = Tm.f[f];
                auto others = [&](int i) -> double {
                    double pr = Tm.coef ? Tm.coef[i] : 1.0;
                    for (int f2 = 0; f2 < Tm.n_factors; ++f2)
                        if (f2 != f) pr *= ir_factor(Tm.f[f2], x, i);
                    return pr;
                };
                if (!Fc.idx && Fc.size == 1) {  // scalar target: team reduction over the observations
                    double a = 0.0;
                    for (int i = tid; i < N; i += TS) a = fma(r[i], others(i), a);
                    a = team_sum<W>(a, tid, red);
                    if (tid == 0) g_s[Fc.offset] += a;
                } else if (!Fc.idx) {  // elementwise target (vector variable of the block's length)
                    for (int i = tid; i < N; i += TS) g_s[Fc.offset + i] += r[i] * others(i);
                } else {  // indexed target: pull through the CSR transpose of idx (fixed order)
                    for (int j = tid; j < Fc.size; j += TS) {
                        double a = 0.0;
                        for (int e = Fc.rowptr[j]; e < Fc.rowptr[j + 1]; ++e) {
                            const int i = Fc.rowobs[e];
                            a = fma(r[i], others(i), a);
                        }
                        g_s[Fc.offset + j] += a;
                    }
                }
                team_sync<W>();
            }
        }
    }

    template <int NPL, int W, bool SMALL = false>
    __device__ __noinline__ static double eval(const Params& P, const char* s, const double* q_s, double* g_s, int tid, double* red) {
        return eval_impl<NPL, W, false>(P, s, q_s, g_s, tid, red);
    }

    template <int NPL, int W, bool EXTENDED>
    __device__ __forceinline__ static double eval_impl(const Params& P, const char*, const double* q_s, double* g_s, int tid,
                                                       double* red) {
        constexpr int TS = 32 * W;
        const int slot = (W == 1) ? (int)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) : (int)blockIdx.x;
        double* x = P.scratch + (long long)slot * P.stride;
        double* r = x + P.n_pad;
        const int n = P.n;
        double lp = 0.0;  // per-thread partial; reduced once at the end

        // ---- 1. constrain (+ log-Jacobians); gx accumulates in g_s -----------------------------------------------------
        for (int v = 0; v < P.n_vars; ++v) {
            const IrVarD V = P.vars[v];
            if constexpr (EXTENDED) {
                if (ir_extended_transforms(V.transform)) {  // uniform branch: a prefix sum or a softmax, on one thread
                    if (tid == 0)
                        lp += V.transform == B200_IR_T_SIMPLEX ? ir_simplex_forward(P.vars + v, q_s, x) : ir_ordered_forward(P.vars + v, q_s, x);
                    for (int j = tid; j < V.size; j += TS) g_s[V.offset + j] = 0.0;
                    continue;
                }
            }
            for (int j = tid; j < V.size; j += TS) {
                const int i = V.offset + j;
                x[i] = ir_backward(V, q_s[i], lp);
                g_s[i] = 0.0;
            }
        }
        team_sync<W>();

        // ---- 2a. priors ---------------------------------------------------------------------------------------------
        for (int k = 0; k < P.n_priors; ++k) {
            const IrPriorD F = P.priors[k];
            if (F.dist == B200_IR_P_FLAT) continue;
            if constexpr (EXTENDED) {
                if (F.dist == B200_IR_P_DIRICHLET) {  // uniform branch: out of line, on one thread
                    if (tid == 0) lp += ir_dirichlet(P.priors + k, x);
                    team_sync<W>();
                    continue;
                }
                if (F.dist == B200_IR_P_INVERSEGAMMA) {  // uniform branch: out of line
                    lp += ir_inversegamma(P.priors + k, x, g_s, tid, TS);
                    team_sync<W>();
                    continue;
                }
            }
            const double a0 = par(F.p[0], x), a1 = par(F.p[1], x), a2 = par(F.p[2], x);
            double s[3] = {0.0, 0.0, 0.0};  // sums for the parameter gradients
            for (int j = tid; j < F.size; j += TS) {
                const int i = F.offset + j;
                const double xv = x[i];
                double gxi = 0.0;
                switch (F.dist) {
                    case B200_IR_P_NORMAL: {  // continuous.py:526-527
                        const double z = (xv - a0) / a1;
                        lp += -0.5 * z * z + F.c0 - log(a1);
                        gxi = -z / a1; s[0] += z / a1; s[1] += (z * z - 1.0) / a1;
                    } break;
                    case B200_IR_P_HALFNORMAL: {  // continuous.py:909-911
                        const double z = xv / a0;
                        lp += -0.5 * z * z + F.c0 - log(a0);
                        gxi = -z / a0; s[0] += (z * z - 1.0) / a0;
                    } break;
                    case B200_IR_P_CAUCHY: {  // continuous.py:2287-2288
                        const double u = xv - a0, den = a1 * a1 + u * u, t = u / a1;
                        lp += F.c0 - log(a1) - log1p(t * t);
                        gxi = -2.0 * u / den; s[0] += 2.0 * u / den; s[1] += (u * u - a1 * a1) / (a1 * den);
                    } break;
                    case B200_IR_P_HALFCAUCHY: {  // continuous.py:2383-2385
                        const double den = a0 * a0 + xv * xv, t = xv / a0;
                        lp += F.c0 - log(a0) - log1p(t * t);
                        gxi = -2.0 * xv / den; s[0] += (xv * xv - a0 * a0) / (a0 * den);
                    } break;
                    case B200_IR_P_EXPONENTIAL:  // continuous.py:1478-1480 (mu = 1 / lam)
                        lp += log(a0) - a0 * xv;
                        gxi = -a0; s[0] += 1.0 / a0 - xv;
                        break;
                    case B200_IR_P_STUDENTT: {  // continuous.py:1936-1944; a0 = nu (constant), a1 = mu, a2 = sigma
                        const double z = (xv - a1) / a2;
                        lp += F.c0 - log(a2) - 0.5 * (a0 + 1.0) * log1p(z * z / a0);
                        const double w = (a0 + 1.0) * z / (a2 * (a0 + z * z));
                        gxi = -w; s[1] += w; s[2] += -1.0 / a2 + w * z;
                    } break;
                    case B200_IR_P_UNIFORM: lp += F.c0; break;  // continuous.py:309-314
                    case B200_IR_P_GAMMA:  // continuous.py:2512-2515
                        lp += F.c0 + (a0 - 1.0) * log(xv) - a1 * xv;
                        gxi = (a0 - 1.0) / xv - a1;
                        break;
                    case B200_IR_P_BETA:  // continuous.py:1250-1256
                        lp += F.c0 + (a0 - 1.0) * log(xv) + (a1 - 1.0) * log1p(-xv);
                        gxi = (a0 - 1.0) / xv - (a1 - 1.0) / (1.0 - xv);
                        break;
                    case B200_IR_P_LOGNORMAL: {  // continuous.py:1807-1814
                        const double lx = log(xv), z = (lx - a0) / a1;
                        lp += -0.5 * z * z - lx + F.c0 - log(a1);
                        gxi = (-z / a1 - 1.0) / xv; s[0] += z / a1; s[1] += (z * z - 1.0) / a1;
                    } break;
                    default: break;
                }
                g_s[i] += gxi;
            }
            const bool any_ref = F.p[0].kind | F.p[1].kind | F.p[2].kind;
            if (any_ref) {  // uniform branch: the descriptor is the same for every thread
                team_sync<W>();
                team_sum_n<W>(s, tid, red);
                if (tid == 0) {
#pragma unroll
                    for (int a = 0; a < 3; ++a)
                        if (F.p[a].kind) g_s[F.p[a].ref] += s[a];
                }
            }
            team_sync<W>();
        }

        if constexpr (EXTENDED) {
            const int n_spec = ir_spec_count(P.terms);
            if (n_spec) {  // uniform branch: the spectral terms' rows, before any likelihood reads them
                ir_spectral_forward(ir_specs(P.terms, n_spec), n_spec, x, tid, TS);
                team_sync<W>();
            }
        }

        // ---- 2b. likelihoods: eta_i = sum_t coef_t[i] prod_f x_f[idx_f[i]] ----------------------------------------------
        for (int l = 0; l < P.n_liks; ++l) {
            const IrLikD L = P.liks[l];
            const int N = (int)L.N;
            const double sg_s = ir_slot(L, x);
            const bool zi = EXTENDED && ir_zi_liks(L.dist);  // zero-inflated / hurdle
            const bool gamma = L.dist == B200_IR_L_GAMMA_LOG || (EXTENDED && L.dist == B200_IR_L_HURDLE_GAMMA);
            const bool disp = L.dist == B200_IR_L_NEGBINOMIAL_LOG || gamma ||  // sg_s is the dispersion alpha
                              (EXTENDED && (L.dist == B200_IR_L_ZERO_INFLATED_NEGATIVE_BINOMIAL || L.dist == B200_IR_L_HURDLE_NEGATIVE_BINOMIAL));
            const double la = disp ? log(sg_s) : 0.0;
            double s_sig = 0.0, s_psi = 0.0;
            const bool ordinal = EXTENDED && ir_ordinal_liks(L.dist);
            const bool mixture = EXTENDED && ir_mixture_liks(L.dist);
            const bool beta = EXTENDED && ir_beta_liks(L.dist);
            const bool bounded = EXTENDED && (ordinal || zi || mixture || beta || ir_bounded_liks(L.dist) || ir_survival_liks(L.dist));
            if constexpr (EXTENDED) {
                if (mixture) {  // uniform branch: out of line, with the per-component gradients
                    lp += ir_mixture_pass<W>(P.liks + l, P.terms, x, r, x + P.ord_row, g_s, tid, red);
                } else if (beta) {  // uniform branch: out of line, with the phi-only terms of a random phi
                    const IrPartials b = ir_beta_pass<W>(P.liks + l, P.terms, x, r, sg_s, tid);
                    lp += b.lp;
                    s_sig = b.s_sig;
                } else if (zi) {  // uniform branch: out of line
                    const IrZiPartials b = ir_zi_pass<W>(P.liks + l, P.terms, x, r, x + P.ord_row, sg_s, la, tid);
                    lp += b.lp;
                    s_sig = b.s_a;
                    s_psi = b.s_psi;
                } else if (bounded) {  // uniform branch: out of line
                    const IrPartials b = ordinal ? ir_ordinal_pass<W>(P.liks + l, P.terms, x, r, x + P.ord_row, sg_s, tid)
                                                 : ir_bounded_pass<W>(P.liks + l, P.terms, x, r, sg_s, tid);
                    lp += b.lp;
                    s_sig = b.s_sig;
                }
            }
            if (!bounded) for (int i = tid; i < N; i += TS) {
                const double eta = ir_eta(P.terms, L.term0, L.n_terms, x, i, N);
                const double yi = L.yoff >= 0 ? x[L.yoff + i] : L.y[i];
                const double ri = ir_base_term(L, i, yi, eta, sg_s, la, lp, s_sig);
                r[i] = ri;
                if (L.yoff >= 0) g_s[L.yoff + i] -= ri;  // this thread owns element i of the latent variable
            }
            if (disp && L.sigma_kind == B200_IR_S_REF) {  // uniform branch: the alpha-dependent normalising terms
                const double a = sg_s;
                const IrLikD& Lt = P.liks[l];  // read here, not kept live through the observation loop
                if (gamma) {
                    if (tid == 0) {
                        const double sly = Lt.sum_log_y;
                        const double Ny = (EXTENDED && L.dist == B200_IR_L_HURDLE_GAMMA) ? (double)Lt.n_tab : (double)N;  // hurdle_gamma: N+
                        lp += Ny * (a * la - lgamma(a)) + (a - 1.0) * sly;
                        s_sig += Ny * (la + 1.0 - digamma(a)) + sly;
                    }
                } else if (a <= kNegBinPoissonAlpha) {
                    // sum_i lgamma(y_i + a) - lgamma(a) over the distinct values: team-strided, fixed order
                    const double lga = lgamma(a), pa = digamma(a);
                    const double* tu = Lt.tab_u;
                    const double* tc = Lt.tab_cnt;
                    const int n_tab = Lt.n_tab;
                    for (int k = tid; k < n_tab; k += TS) {
                        const double u = tu[k], c = tc[k];
                        lp = fma(c, lgamma(u + a) - lga, lp);
                        s_sig = fma(c, digamma(u + a) - pa, s_sig);
                    }
                }
            }
            if (tid == 0) lp += L.c0;
            team_sync<W>();
            if constexpr (EXTENDED) {
                if (ordinal && P.terms[L.term0 + L.n_terms].n_factors) {  // uniform branch: variable cutpoints
                    ir_cutpoint_grad<W>(P.liks + l, P.terms, r, x + P.ord_row, g_s, tid);
                    team_sync<W>();
                }
                if (zi) {  // uniform branch: the psi block's gradient
                    const IrTermD* pt = P.terms + L.term0 + L.n_terms;
                    if (L.nu > 0.0) {  // the terms of logit(psi), fed the zeta row
                        term_grad<W, true>(P, L.term0 + L.n_terms, (int)L.nu, x + P.ord_row, N, x, g_s, tid, red);
                    } else if (pt->n_factors) {  // a psi variable: one team reduction
                        const double tot = team_sum<W>(s_psi, tid, red);
                        if (tid == 0) g_s[pt->f[0].offset] += tot;
                        team_sync<W>();
                    }
                }
            }
            if (L.sigma_kind == B200_IR_S_REF) {
                const double tot = team_sum<W>(s_sig, tid, red);
                if (tid == 0) g_s[L.sigma.ref] += tot;
                team_sync<W>();
            }
            // gradient of every (term, factor) of the predictor: d eta_i / d x_f = coef * (other factors)
            term_grad<W, EXTENDED>(P, L.term0, L.n_terms, r, N, x, g_s, tid, red);
        }
        if constexpr (EXTENDED) {
            const int n_spec = ir_spec_count(P.terms);
            if (n_spec) {  // uniform branch: the spectral terms' g_b rows back to z, a and l
                ir_spectral_grad<W>(ir_specs(P.terms, n_spec), n_spec, x, g_s, tid, red);
                team_sync<W>();
            }
        }

        // ---- 2c. AR(1): h_0 ~ Normal(0, init_sigma), h_t - phi h_{t-1} ~ Normal(0, sigma)  (timeseries.py:646-676) ------
        for (int k = 0; k < P.n_ar1; ++k) {
            const IrAr1D A = P.ar1[k];
            const double phi = par(A.phi, x), sg = par(A.sigma, x);
            const double i2 = 1.0 / (sg * sg);
            const double* h = x + A.offset;
            double s[2] = {0.0, 0.0};  // sum e h_{t-1}, sum e^2
            for (int t = tid; t < A.size; t += TS) {
                const double ht = h[t];
                double g = 0.0;
                if (t >= 1) {
                    const double hm = h[t - 1], e = ht - phi * hm;
                    g -= e * i2;
                    s[0] = fma(e, hm, s[0]);
                    s[1] = fma(e, e, s[1]);
                } else {
                    const double zi = ht / A.init_sigma;
                    g -= zi / A.init_sigma;
                    lp += -0.5 * zi * zi - B200_HALF_LOG_2PI - log(A.init_sigma);
                }
                if (t + 1 < A.size) g = fma(phi * i2, h[t + 1] - phi * ht, g);
                g_s[A.offset + t] += g;
            }
            team_sync<W>();
            team_sum_n<W>(s, tid, red);
            if (tid == 0) {
                lp += -0.5 * s[1] * i2 - (A.size - 1) * (B200_HALF_LOG_2PI + log(sg));
                if (A.phi.kind) g_s[A.phi.ref] += s[0] * i2;
                if (A.sigma.kind) g_s[A.sigma.ref] += (s[1] * i2 - (double)(A.size - 1)) / sg;
            }
            team_sync<W>();
        }

        // ---- 3. chain rule through the transforms -------------------------------------------------------------------------
        for (int v = 0; v < P.n_vars; ++v) {
            const IrVarD V = P.vars[v];
            if (V.transform == B200_IR_T_NONE) continue;
            if constexpr (EXTENDED) {
                if (ir_extended_transforms(V.transform)) {  // uniform branch: a reverse prefix sum or the softmax's, on one thread
                    if (tid == 0) {
                        if (V.transform == B200_IR_T_SIMPLEX) ir_simplex_chain(P.vars + v, x, g_s);
                        else ir_ordered_chain(P.vars + v, q_s, g_s);
                    }
                    continue;
                }
            }
            for (int j = tid; j < V.size; j += TS) {
                const int i = V.offset + j;
                const double xv = x[i];
                if (V.transform == B200_IR_T_LOG) {
                    g_s[i] = fma(g_s[i], xv, 1.0);
                } else {
                    // dx/dz = (hi - lo) s (1 - s), s = sigmoid(z), in the form e / (1 + e)^2 with e = exp(-|z|): s recovered
                    // from x, or 1 - s, cancels at large |z| (relative error 1e-3 at |z| = 30)
                    const double sg = (xv - V.lo) / (V.hi - V.lo);
                    const double e = exp(-fabs(q_s[i]));
                    g_s[i] = fma(g_s[i], (V.hi - V.lo) * (e / ((1.0 + e) * (1.0 + e))), 1.0 - 2.0 * sg);
                }
            }
        }
        for (int i = n + tid; i < TS * NPL; i += TS) g_s[i] = 0.0;  // padding of the state vectors
        team_sync<W>();
        return team_sum<W>(lp, tid, red);
    }
};

struct IrExtendedModel : IrModel {
    template <int NPL, int W, bool SMALL = false>
    __device__ __noinline__ static double eval(const Params& P, const char* s, const double* q_s, double* g_s, int tid, double* red) {
        return eval_impl<NPL, W, true>(P, s, q_s, g_s, tid, red);
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// Pointwise log-likelihood of one likelihood factor for a batch of (unconstrained) draws: out[d][i] = log p(y_i | draw d).
// What pm.compute_log_likelihood evaluates per draw through a compiled function (pymc/stats/log_density.py:31-77,
// :129-195) -- the `log_likelihood` group LOO / WAIC need.  One warp per draw; the constrained values go through the
// team scratch slice like in eval().  Elementwise constants (log 2pi, lgamma) are included, unlike in eval() where they are
// folded into one constant per factor.
// ---------------------------------------------------------------------------------------------------------------------

// log p(y_i | eta) of observation i with every constant, through the term function eval's pass uses: a base family's
// term plus ir_obs_const; a zero-inflated / hurdle count's plus that of f at y > 0; a censored / truncated Normal's plus
// -log(2 pi) / 2 except at a censoring bound, a LogNormal's plus -log(2 pi) / 2 - log y_i there; an ordinal or Weibull
// one's has none.
template <bool EXTENDED>  // as IrModel / IrExtendedModel
__device__ __forceinline__ double ir_obs_loglik(const IrLikD& L, const IrTermD* terms, const double* x, int i, double eta,
                                                double sg_s, double la) {
    const double y = L.y[i];
    if (EXTENDED && ir_mixture_liks(L.dist)) {
        const double lse = ir_mix_obs(L.dist, (int)L.nu, ir_mix_block(L, terms, x, nullptr), y, eta).lse;
        return lse - (L.dist == B200_IR_L_NORMAL_MIXTURE ? B200_HALF_LOG_2PI : lgamma(y + 1.0));
    }
    if (EXTENDED && ir_zi_liks(L.dist)) {
        const IrPsi ps = ir_psi(terms + L.term0 + L.n_terms, (int)L.nu, x, i, (int)L.N);
        const double lp = ir_zi_term(L.dist, y, eta, ir_scale(L, i, sg_s), sg_s, la, ps).lp;
        return y > 0.0 ? lp + ir_obs_const(L, i, y, sg_s, la) : lp;
    }
    if (EXTENDED && ir_ordinal_liks(L.dist)) {
        const double s = ir_scale(L, i, L.sigma_kind == B200_IR_S_NONE ? 1.0 : sg_s);  // the logistic link: s = 1
        return ir_ordinal_term(L, terms[L.term0 + L.n_terms], x, i, eta, s).lp;
    }
    if (EXTENDED && ir_weibull_liks(L.dist)) return ir_weibull_term(L, i, eta, sg_s, la).lp;
    if (EXTENDED && ir_beta_liks(L.dist)) return ir_beta_term(L, i, eta, sg_s).lp + ir_beta_const(L, i, sg_s);
    if (EXTENDED && (ir_bounded_liks(L.dist) || ir_survival_liks(L.dist))) {
        const bool at_bound = L.cens && L.cens[i] != 0;
        const double ly = ir_bounded_liks(L.dist) ? 0.0 : y;  // a LogNormal's y is log y_i
        return ir_bounded_term(L, i, eta, ir_scale(L, i, sg_s)).lp - (at_bound ? 0.0 : B200_HALF_LOG_2PI + ly);
    }
    double lp = 0.0, s_sig = 0.0;
    ir_base_term(L, i, y, eta, sg_s, la, lp, s_sig);
    return lp + ir_obs_const(L, i, y, sg_s, la);
}

template <bool EXTENDED>
__global__ void __launch_bounds__(256) ir_pointwise_kernel(const IrModel::Params P, int lik, long long D,
                                                           const double* __restrict__ draws /*[D][n]*/,
                                                           double* __restrict__ out /*[D][N]*/) {
    const int lane = threadIdx.x & 31;
    const int slot = (int)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5));
    double* x = P.scratch + (long long)slot * P.stride;
    const IrLikD& L = P.liks[lik];
    const int N = (int)L.N, n = P.n;
    const long long stride = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long d = slot; d < D; d += stride) {
        const double* q = draws + d * n;
        for (int v = 0; v < P.n_vars; ++v) {
            const IrVarD V = P.vars[v];
            if constexpr (EXTENDED) {
                if (ir_extended_transforms(V.transform)) {
                    if (lane == 0) {
                        if (V.transform == B200_IR_T_SIMPLEX) ir_simplex_forward(P.vars + v, q, x);
                        else ir_ordered_forward(P.vars + v, q, x);
                    }
                    continue;
                }
            }
            double lj = 0.0;  // the log-Jacobian is not part of the likelihood
            for (int j = lane; j < V.size; j += 32) x[V.offset + j] = ir_backward(V, q[V.offset + j], lj);
        }
        __syncwarp();
        if constexpr (EXTENDED) {
            const int n_spec = ir_spec_count(P.terms);
            if (n_spec) {
                ir_spectral_forward(ir_specs(P.terms, n_spec), n_spec, x, lane, 32);
                __syncwarp();
            }
        }
        const double sg_s = ir_slot(L, x), la = log(sg_s);  // la: log alpha, read only by the families with a dispersion
        for (int i = lane; i < N; i += 32) {
            const double eta = ir_eta(P.terms, L.term0, L.n_terms, x, i, N);
            out[d * N + i] = ir_obs_loglik<EXTENDED>(L, P.terms, x, i, eta, sg_s, la);
        }
        __syncwarp();
    }
}

}  // namespace b200
