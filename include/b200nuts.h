/*
 * b200nuts.h -- C ABI of the B200-native NUTS/HMC engine (libb200nuts.so).
 *
 * This is the drop-in boundary for ONE hot path of pymc-devs/pymc:
 *     model.logp_dlogp_function  evaluated inside  CpuLeapfrogIntegrator.step  under  NUTS._build_tree.
 * The reference has no C API (it is pure Python); every entry point below cites the Python
 * interface it replaces.  Host bindings are plain ctypes (pymc_b200/_lib.py); INTEGRATION.md shows
 * the reference-side shim a maintainer would add.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no C++/torch types cross the boundary.
 *   - every function returns 0 on success, <0 on failure; b200_last_error() gives the message
 *     (thread-local).  No exception crosses the ABI.  B200_E_SHAPE (below) marks one refusal that
 *     a caller may route around.
 *   - NUMERICAL failures are not errors: a non-finite energy inside a trajectory is a divergence
 *     recorded per chain/draw in the stats (reference: IntegrationError -> divergence,
 *     hmc/integration.py:95-107, hmc/nuts.py:399-440); a non-finite energy at the START of a draw
 *     ("Bad initial energy", hmc/base_hmc.py:205-224) freezes that chain and sets its
 *     bad_energy flag -- the host wrapper raises SamplingError like the reference.
 *   - the caller owns every input/output buffer.  Each call states whether its pointers are host
 *     or device memory via `B200_MEM_HOST` / `B200_MEM_DEVICE`; host buffers are staged
 *     through pinned memory inside the call.
 *   - a handle is bound to the CUDA device that was current at creation and is not thread-safe
 *     (one process per GPU; the reference isolates chains in processes, sampling/parallel.py).
 *   - all floating point is IEEE fp64, like the reference's floatX=float64 default.
 */
#ifndef B200NUTS_H
#define B200NUTS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200NUTS_VERSION 300 /* 0.3.0: B200_MASS_DENSE_ADAPT (b200_nuts_cfg.mass_update_window / .adaptation_window_multiplier,
                              * b200_chain_summary.final_cov); 0.2.0: b200_model_desc.ir (ModelSpec IR) */

/* b200_model_create: the hand-written kernel of the model kind cannot run this size or data layout (EIGHT_SCHOOLS and
 * RADON: n > 256, the chain-per-warp limit; RADON: padded observation rows that do not fit 227 KB of shared memory in the
 * logp launch or in the NUTS launch with no tree level in shared memory).  The same model written as B200_MODEL_IR runs on
 * the generic device function.  Every other failure returns -1. */
#define B200_E_SHAPE (-2)

/* memory space of caller-provided buffers */
#define B200_MEM_HOST 0
#define B200_MEM_DEVICE 1

/* model kinds: the hand-written fused logp+gradient device functions (csrc/models.cuh).
 * Each replaces the compiled PyTensor callable built at pymc/model/core.py:232-267 for that model. */
#define B200_MODEL_STD_NORMAL 0    /* x ~ Normal(0,1)^n                           (test model)      */
#define B200_MODEL_EIGHT_SCHOOLS 1 /* BASELINE config 1, q = [mu, log tau, theta_t[J]]              */
#define B200_MODEL_RADON 2         /* BASELINE config 2, benchmarks/benchmarks/benchmarks.py:26-46  */
#define B200_MODEL_LOGISTIC 3      /* BASELINE config 3, beta~N(0,1), y~Bernoulli(logit_p=X beta)   */
#define B200_MODEL_STOCHVOL 4      /* BASELINE config 4, AR(1) stochastic volatility               */
#define B200_MODEL_MVGAUSS 5       /* BASELINE config 5, x~MvNormal(0, chol=L), dense mass matrix   */
#define B200_MODEL_IR 6            /* any model of the closed factor set below (b200_ir): ONE generic fused logp+gradient
                                    * device function (csrc/ir_model.cuh), no new CUDA per model.  The kinds above are
                                    * hand-specialised fast paths that pymc_b200.ir.specialise() routes matching IR to. */

/* ---- ModelSpec IR: what Model.logp_dlogp_function closes over, as data --------------------------------------------------
 * Ordered value variables with their transforms (pymc/logprob/transforms.py:880-891 log, :1026-1073 interval), and a list
 * of factors whose log-densities are summed (pymc/model/core.py:688-690).  All pointers are HOST memory, copied at create.
 * Parameters are constants or SCALAR value variables seen through their transform (hierarchical priors). */
#define B200_IR_T_NONE 0
#define B200_IR_T_LOG 1
#define B200_IR_T_INTERVAL 2
/* Ordered (transforms.py:79-120), ascending: x_0 = z_0 (ORDERED_POSITIVE: exp z_0), x_k = x_{k-1} + exp z_k; log|J| =
 * sum_{k>=1} z_k (ORDERED_POSITIVE: sum_k z_k).  Not elementwise: the draws of a model with such a variable are constrained
 * on the host.  An ordered variable takes only real-line priors (flat, normal, studentt, cauchy, or a latent normal /
 * studentt); ORDERED_POSITIVE also counts as positive support. */
#define B200_IR_T_ORDERED 3
#define B200_IR_T_ORDERED_POSITIVE 4
/* Simplex (transforms.py:1091-1116): a variable of size K - 1 whose constrained value is the K weights
 * w = softmax([z, -sum z]); log|J| = log K + sum_k log w_k.  It carries exactly one prior, a DIRICHLET of length K, and is
 * used only as the weights of a NORMAL_MIXTURE / POISSON_MIXTURE (never as a parameter, a term factor, cutpoints, psi, an
 * AR(1) variable or a latent factor).  The draws of a model with such a variable are constrained on the host. */
#define B200_IR_T_SIMPLEX 5
/* prior densities (pymc/distributions/continuous.py): parameters in p[0..2] */
#define B200_IR_P_FLAT 0        /*                       :364-419   */
#define B200_IR_P_NORMAL 1      /* mu, sigma             :526-527   */
#define B200_IR_P_HALFNORMAL 2  /* sigma                 :909-911   */
#define B200_IR_P_CAUCHY 3      /* alpha, beta           :2287-2288 */
#define B200_IR_P_HALFCAUCHY 4  /* beta                  :2383-2385 */
#define B200_IR_P_EXPONENTIAL 5 /* lam                   :1478-1480 */
#define B200_IR_P_STUDENTT 6    /* nu (const), mu, sigma :1936-1944 */
#define B200_IR_P_UNIFORM 7     /* lower, upper (const)  :309-314   */
#define B200_IR_P_GAMMA 8       /* alpha, beta (const)   :2512-2515 */
#define B200_IR_P_BETA 9        /* alpha, beta (const)   :1250-1256 */
#define B200_IR_P_LOGNORMAL 10  /* mu, sigma             :1807-1814 */
#define B200_IR_P_DIRICHLET 11  /* a (const), the concentration of every one of the K components; only on a SIMPLEX
                                 * variable of size K - 1    multivariate.py:557-585 */
#define B200_IR_P_INVERSEGAMMA 12 /* alpha, beta (const > 0); positive support   :2631-2640 */
/* likelihoods of a linear predictor eta_i = sum_t coef_t[i] * prod_f x_f[idx_f[i]] */
#define B200_IR_L_NORMAL 0          /* y ~ Normal(eta, sigma)                    continuous.py:526-527  */
#define B200_IR_L_BERNOULLI_LOGIT 1 /* y ~ Bernoulli(logit_p = eta)              discrete.py:362-367    */
#define B200_IR_L_POISSON_LOG 2     /* y ~ Poisson(exp(eta))                     discrete.py:581-586    */
#define B200_IR_L_STUDENTT 3        /* y ~ StudentT(nu, eta, sigma)              continuous.py:1936-1944 */
#define B200_IR_L_NORMAL_LOGVAR 4   /* y ~ Normal(0, exp(eta / 2))                                      */
/* The three families below carry their parameter in the likelihood's `sigma` slot:
 *   BINOMIAL_LOGIT     trials n: CONST (sigma.value) or OBS (sigma_obs[N]), integer >= 0; integer 0 <= y <= n
 *   NEGBINOMIAL_LOG    dispersion alpha: CONST (> 0) or REF (a scalar variable with positive support); integer y >= 0.
 *                      Above alpha = 1e10 the density is the Poisson(exp(eta)) limit, as in the reference.
 *   GAMMA_LOG          shape alpha: CONST (> 0) or REF; y > 0                                                        */
#define B200_IR_L_BINOMIAL_LOGIT 5  /* y ~ Binomial(n, logit_p = eta)            discrete.py:141-152    */
#define B200_IR_L_NEGBINOMIAL_LOG 6 /* y ~ NegativeBinomial(mu = exp(eta), alpha) discrete.py:700-745   */
#define B200_IR_L_GAMMA_LOG 7       /* y ~ Gamma(alpha, beta = alpha exp(-eta))  continuous.py:2478-2521 */
/* Normal observations measured with bounds.  For these two dists `y` points at a [3][N] block: row 0 is y, row 1 the lower
 * bound, row 2 the upper bound of each observation, -inf / +inf where that side is open.  sigma as for NORMAL (CONST, REF
 * or OBS).
 *   CENSORED_NORMAL   pm.Censored(Normal(eta, sigma), lower, upper): log Phi(z) where y_i == lower_i, log(1 - Phi(z)) where
 *                     y_i == upper_i, the Normal density elsewhere, z = (y_i - eta_i) / sigma
 *   TRUNCATED_NORMAL  pm.TruncatedNormal(eta, sigma, lower, upper): the Normal density minus log(Phi(b) - Phi(a)) of the
 *                     standardised bounds (a one-sided form where one side is open) */
#define B200_IR_L_CENSORED_NORMAL 8  /* logprob/censoring.py:213-248 over Normal; dist_math.py:126-142 */
#define B200_IR_L_TRUNCATED_NORMAL 9 /* TruncatedNormal.logp continuous.py:720-747; dist_math.py:126-182 */
/* Ordinal observations y_i in 0..K-1 with K - 1 cutpoints c: log(F(b) - F(a)), a = (c_{y-1} - eta) / s,
 * b = (c_y - eta) / s, c_{-1} = -inf, c_{K-1} = +inf; F the logistic CDF (s = 1) or the standard Normal one.
 *   nu             K >= 2
 *   terms[n_terms] the cutpoint term, one past the predictor's: one unindexed factor on a variable of size K - 1 (ordered
 *                  unless K = 2), or n_factors = 0 and coef = the K - 1 constants, finite and strictly increasing
 *   sigma          ORDERED_LOGISTIC: NONE; ORDERED_PROBIT: as for NORMAL (CONST, REF or OBS) */
#define B200_IR_L_ORDERED_LOGISTIC 10 /* pm.OrderedLogistic discrete.py:1231-1326 as Categorical.logp :1190-1206 */
#define B200_IR_L_ORDERED_PROBIT 11   /* pm.OrderedProbit discrete.py:1329-1432 as Categorical.logp :1190-1206   */
/* Zero-inflated and hurdle observations with mixing probability psi, the probability of the count / positive component f
 * (the family of the same name above at eta; P0 = f(0)):
 *   ZERO_INFLATED_*  y = 0: log((1 - psi) + psi P0);  y > 0: log psi + log f(y)
 *   HURDLE_*         y = 0: log(1 - psi);             y > 0: log psi + log f(y) - log(1 - P0)  (HURDLE_GAMMA: no division)
 *   terms[n_terms ..] the psi block, one past the predictor's terms; nu says its form:
 *                  nu = 0      one term, psi itself: n_factors = 0 and coef = the one constant, 0 < psi < 1; or one unindexed
 *                              factor on a scalar variable with an INTERVAL inside [0, 1] and coef = NULL
 *                  nu = m >= 1 psi_i = sigmoid(zeta_i), zeta_i the sum of the m terms terms[n_terms .. n_terms + m), of any kind
 *   sigma          the family's slot: NONE (Poisson), trials as for BINOMIAL_LOGIT, alpha as for NEGBINOMIAL_LOG / GAMMA_LOG
 *   y              integers >= 0 (ZERO_INFLATED_BINOMIAL: <= n); HURDLE_GAMMA: finite and >= 0.  y_var must be 0. */
#define B200_IR_L_ZERO_INFLATED_POISSON 12           /* pm.ZeroInflatedPoisson mixture.py:577-638           */
#define B200_IR_L_ZERO_INFLATED_BINOMIAL 13          /* pm.ZeroInflatedBinomial mixture.py:641-702          */
#define B200_IR_L_ZERO_INFLATED_NEGATIVE_BINOMIAL 14 /* pm.ZeroInflatedNegativeBinomial mixture.py:705-802  */
#define B200_IR_L_HURDLE_POISSON 15                  /* pm.HurdlePoisson mixture.py:873-922                 */
#define B200_IR_L_HURDLE_NEGATIVE_BINOMIAL 16        /* pm.HurdleNegativeBinomial mixture.py:925-978        */
#define B200_IR_L_HURDLE_GAMMA 17                    /* pm.HurdleGamma mixture.py:981-1034                  */
/* Survival (time-to-event) observations y > 0 with a log link.  With u = log y - eta and t(y) = exp(alpha u) = (y / beta)^alpha:
 *   WEIBULL_LOG        y ~ Weibull(alpha, beta = exp(eta)): log f = log alpha - eta + (alpha - 1) u - t.  The Exponential
 *                      with scale exp(eta) is alpha = 1.  sigma: alpha, CONST (> 0) or REF (a scalar of positive support).
 *   LOGNORMAL          y ~ LogNormal(mu = eta, sigma): the Normal of log y at (eta, sigma), minus log y.  sigma as for NORMAL.
 *   CENSORED_*         `y` is the [3][N] block (y, lower, upper) of CENSORED_NORMAL: log F(y) where y_i == lower_i (Weibull:
 *                      log(1 - e^-t); LogNormal: log Phi of log y), log S(y) where y_i == upper_i (-t; log(1 - Phi)), the
 *                      density elsewhere
 *   TRUNCATED_*        the same block: the density minus log(S(lower) - S(upper)), a one-sided form where a side is open
 * y finite and > 0; lower >= 0 or -inf and upper > 0 or +inf, where lower 0 / -inf and upper +inf are open sides;
 * lower_i < upper_i and lower_i <= y_i <= upper_i; a truncated factor has a finite lower bound > 0 or a finite upper bound.
 * nu is unused.  y_var must be 0. */
#define B200_IR_L_WEIBULL_LOG 18            /* pm.Weibull continuous.py:2740-2831; pm.Exponential :1461-1480 */
#define B200_IR_L_LOGNORMAL 19              /* pm.LogNormal continuous.py:1723-1846                          */
#define B200_IR_L_CENSORED_WEIBULL_LOG 20   /* pm.Censored(pm.Weibull.dist(...)) logprob/censoring.py:213-248 */
#define B200_IR_L_CENSORED_LOGNORMAL 21     /* pm.Censored(pm.LogNormal.dist(...))                            */
#define B200_IR_L_TRUNCATED_WEIBULL_LOG 22  /* pm.Truncated(pm.Weibull.dist(...)) truncated.py                */
#define B200_IR_L_TRUNCATED_LOGNORMAL 23    /* pm.Truncated(pm.LogNormal.dist(...))                           */
/* Finite mixtures of K >= 2 components: log p(y_i) = logsumexp_k(log w_k + log f_k(y_i))  (mixture.py:469-494)
 *   NORMAL_MIXTURE     f_k = Normal(eta_i + mu_k, sigma_k); y finite
 *   POISSON_MIXTURE    f_k = Poisson(lam_k exp(eta_i)); y integers >= 0
 *   nu             K
 *   n_terms        the predictor's terms, which may be none (eta = 0)
 *   terms[n_terms]     the weights: one unindexed factor on a SIMPLEX variable of size K - 1, or n_factors = 0 and coef = K
 *                      constants, finite, >= 0, summing to 1 (a zero weight drops its component)
 *   terms[n_terms + 1] the components mu_k (Normal) / lam_k (Poisson): one unindexed factor on a variable of size K (Normal:
 *                      no transform or ORDERED; Poisson: positive support), or n_factors = 0 and coef = K constants (finite;
 *                      Poisson: > 0)
 *   terms[n_terms + 2] NORMAL_MIXTURE only, sigma_k: one unindexed factor on a variable of size 1 or K with positive support,
 *                      or n_factors = 0 and coef = K constants > 0
 *   sigma_kind NONE, y_var 0. */
#define B200_IR_L_NORMAL_MIXTURE 24         /* pm.NormalMixture mixture.py:529-546                            */
#define B200_IR_L_POISSON_MIXTURE 25        /* pm.Mixture(w, pm.Poisson.dist(lam, shape=K))                   */
/* Beta regression with a logit mean: mu = sigmoid(eta), precision phi, a = phi mu, b = phi (1 - mu).  sigma: phi, CONST (> 0)
 * or REF (a scalar variable with positive support).  y_var must be 0.
 *   BETA_LOGIT           y ~ Beta(mu, nu = phi): y finite with 0 < y < 1 (0 and 1 are outside the support)
 *   BETA_BINOMIAL_LOGIT  y ~ BetaBinomial(n, a, b): `y` is the [2][N] block (y, trials); trials finite integers >= 0, y an
 *                        integer with 0 <= y <= trials */
#define B200_IR_L_BETA_LOGIT 26             /* pm.Beta(mu, nu) continuous.py:1131-1262, alpha = mu nu :1238-1240 */
#define B200_IR_L_BETA_BINOMIAL_LOGIT 27    /* pm.BetaBinomial discrete.py:178-262                            */
/* The support rule b200_model_create enforces (as ModelIR.validate does): HalfNormal, HalfCauchy, Exponential, Gamma,
 * InverseGamma and LogNormal priors sit on a LOG variable or an INTERVAL with lo >= 0, Beta on an INTERVAL inside [0, 1], Uniform(a, b) on an
 * INTERVAL inside [a, b]; every scale (a prior's sigma / beta / lam, Normal and StudentT sigma including each sigma_obs, an
 * AR(1) sigma, alpha) is a finite constant > 0 or a REF to a scalar of positive support; Poisson y are integers >= 0,
 * Bernoulli y are 0 or 1.  Censored and truncated Normal observations: y finite, lower_i < upper_i, lower never +inf and
 * upper never -inf, lower_i <= y_i <= upper_i; a truncated Normal factor has at least one finite bound. */
#define B200_IR_S_NONE 0
#define B200_IR_S_CONST 1 /* sigma.value               */
#define B200_IR_S_REF 2   /* sigma = x[sigma.ref]      */
#define B200_IR_S_OBS 3   /* sigma_obs[N] (known per-observation scale) */

typedef struct b200_ir_param {
    int32_t kind;  /* 0: constant `value`; 1: the constrained value of the scalar variable at offset `ref` of q */
    int32_t ref;
    double value;
} b200_ir_param;
typedef struct b200_ir_var {
    int32_t offset, size, transform, reserved;
    double lo, hi; /* interval bounds */
} b200_ir_var;
typedef struct b200_ir_prior {
    int32_t dist, var; /* var: index into vars */
    b200_ir_param p[3];
} b200_ir_prior;
typedef struct b200_ir_factor {
    int32_t offset, size; /* the variable's slice of q */
    const int32_t* idx;   /* [N] gather index into the variable, or NULL (scalar: broadcast; size == N: elementwise) */
} b200_ir_factor;
/* A term is coef[i] * prod_f x_f[idx_f[i]] when n_cols == 0.  n_cols > 0 makes it a design term,
 * eta_i += sum_k X[i][k] x[f[0].offset + k]: coef is X, row-major [N][n_cols], finite; n_factors == 1, f[0].size == n_cols
 * and f[0].idx == NULL.  b200_model_create refuses any other design table with the words ModelIR.validate uses.
 *
 * A spectral term (a Hilbert-space approximate GP, pm.gp.HSGP non-centred, hsgp_approx.py:453-473) is a design term with
 * n_factors == 3 whose column weights depend on hyperparameters: eta_i += sum_k Phi[i][k] s_k z_k, with
 *   s_k = a sqrt(S(omega_k; l)),  Q_k = sum_d l_d^2 omega_kd^2  and the power spectral density S of cov (cov.py):
 *   EXPQUAD   S = (2 pi)^(D/2) prod_d l_d exp(-Q/2)
 *   MATERN52  S = 2^D pi^(D/2) Gamma((D+5)/2) 5^(5/2) / (3/4 sqrt(pi)) prod_d l_d (5 + Q)^(-(D+5)/2)
 *   MATERN32  S = 2^D pi^(D/2) Gamma((D+3)/2) 3^(3/2) / (1/2 sqrt(pi)) prod_d l_d (3 + Q)^(-(D+3)/2)
 *   n_cols  M;  f[0] z: a variable of size M, no index, no transform
 *   f[1]    the amplitude a: a scalar variable with positive support (size 1), or size 0 for the constant in the block
 *   f[2]    the lengthscale(s) l: a variable of size 1 (isotropic) or D with positive support, or size 0 for the constants
 *   coef    Phi [N][M] row-major, finite, followed by the block (3 + D + M D doubles):
 *           cov, D, a (> 0; read when f[1].size == 0), l_1 .. l_D (> 0; read when f[2].size == 0), omega [M][D] (finite, >= 0)
 * Such a term may stand wherever a design term may. */
#define B200_IR_COV_EXPQUAD 1
#define B200_IR_COV_MATERN52 2
#define B200_IR_COV_MATERN32 3
typedef struct b200_ir_term {
    const double* coef; /* [N] or NULL (= 1); a design term: X [N][n_cols] */
    int32_t n_factors, n_cols;
    b200_ir_factor f[3];
} b200_ir_term;
/* y_var selects what the factor observes:
 *   0      y[N] is observed data (every zero-initialised table);
 *   v + 1  a LATENT factor: the values are the constrained values of variable v (N == its size; y may be NULL).  This is a
 *          Normal or StudentT prior on variable v whose location is the linear predictor of the terms, e.g. centred group
 *          effects a_j ~ Normal(g0 + g1 u_j + r[region_j], sigma); sigma as above (CONST, REF or OBS: one per element).
 *          The y checks are skipped; b200_pointwise_loglik refuses its index, since it is not a likelihood. */
typedef struct b200_ir_lik {
    int32_t dist, n_terms;
    int64_t N;
    const double* y; /* [N]; [3][N] (y, lower, upper) for the CENSORED_* / TRUNCATED_* dists; [2][N] (y, trials) for
                      * BETA_BINOMIAL_LOGIT; NULL allowed when y_var > 0 */
    const b200_ir_term* terms;
    int32_t sigma_kind, y_var;
    b200_ir_param sigma;
    const double* sigma_obs; /* [N] when sigma_kind == B200_IR_S_OBS (Binomial: trials per observation) */
    double nu;
} b200_ir_lik;
typedef struct b200_ir_ar1 { /* h_0 ~ Normal(0, init_sigma); h_t - phi h_{t-1} ~ Normal(0, sigma)  (timeseries.py:646-676) */
    int32_t var, reserved;
    b200_ir_param phi, sigma;
    double init_sigma;
} b200_ir_ar1;
typedef struct b200_ir {
    int32_t n_vars, n_priors, n_liks, n_ar1;
    const b200_ir_var* vars;
    const b200_ir_prior* priors;
    const b200_ir_lik* liks;
    const b200_ir_ar1* ar1;
} b200_ir;

/* mass-matrix kinds (reference: pymc/step_methods/hmc/quadpotential.py) */
#define B200_MASS_DIAG 0       /* QuadPotentialDiag      :582-630  (fixed diagonal)                   */
#define B200_MASS_DIAG_ADAPT 1 /* QuadPotentialDiagAdapt :211-355  (per-chain Welford windows)        */
#define B200_MASS_DENSE 2      /* QuadPotentialFull      :680-725  (fixed dense covariance)           */
#define B200_MASS_DIAG_ADAPT_GRAD 3 /* QuadPotentialDiagAdaptExp :493-579 with use_grads (init="jitter+adapt_diag_grad",
                                     * pymc/sampling/mcmc.py:1895-1912): var = sqrt(ewvar(draws) / ewvar(gradients));
                                     * persistent engine only */
#define B200_MASS_DENSE_ADAPT 4 /* QuadPotentialFullAdapt :748-845 + _WeightedCovariance :855-907 (init="adapt_full" /
                                 * "jitter+adapt_full", pymc/sampling/mcmc.py:1986-2005): a dense covariance PER CHAIN, estimated
                                 * from the tuning draws in foreground / background windows that grow by
                                 * adaptation_window_multiplier, refreshed (with its Cholesky factor) every mass_update_window
                                 * tuning draws.  Initial covariance = diag(var0) (init_nuts passes the identity), initial mean
                                 * = mean0, initial weight = mass_initial_weight.  Lock-step engine; n <= 1024 */

/* step methods sharing BaseHMC.astep (hmc/base_hmc.py:196-288) */
#define B200_SAMPLER_NUTS 0 /* NUTS._hamiltonian_step          hmc/nuts.py:204-225 */
#define B200_SAMPLER_HMC 1  /* HamiltonianMC._hamiltonian_step hmc/hmc.py:143-200 (+ the uniform(0.85, 1.15) step-size jitter
                             * of hmc.py:35-36, drawn from the chain's step stream); persistent engine only.  Stats: tree_size =
                             * n_steps, mean_tree_accept = accept, index_in_trajectory = n_steps if accepted else 0, depth = 0 */

/* where the momentum noise z ~ N(0,I) of `potential.random()` (quadpotential.py:323-326) comes from */
#define B200_MOMENTUM_DEVICE_PHILOX 0 /* generated on device: Philox4x32-10 + Box-Muller, keyed per chain   */
#define B200_MOMENTUM_HOST_BUFFER 1   /* caller supplies z[C][T][n] (e.g. NumPy Generator.normal: draw-parity) */

typedef struct b200_model b200_model; /* opaque: model constants + observed data resident in HBM */

/* What Model.logp_dlogp_function closes over: the model kind, the raveled size n and the observed
 * data (pymc/model/core.py:464-529).  Unused fields are 0/NULL.  All pointers are HOST memory; the
 * data is copied (and re-laid-out for coalesced access) into device memory by b200_model_create. */
typedef struct b200_model_desc {
    int32_t kind;        /* B200_MODEL_*                                                              */
    int32_t n;           /* length of the raveled unconstrained vector q                              */
    int64_t n_obs;       /* RADON: observations; LOGISTIC: rows; STOCHVOL: T; EIGHT_SCHOOLS: J        */
    int32_t n_groups;    /* RADON: counties                                                           */
    const double* x;     /* RADON: floor[n_obs]; LOGISTIC: X[n_obs][n] row-major; MVGAUSS: prec[n][n]  */
    const double* y;     /* RADON/STOCHVOL/EIGHT_SCHOOLS: y[n_obs]                                     */
    const double* aux;   /* EIGHT_SCHOOLS: sigma[J]; MVGAUSS: cov[n][n] (dense mass matrix)           */
    const int32_t* idx;  /* RADON: county_idx[n_obs] in [0, n_groups)                                 */
    const uint8_t* y_u8; /* LOGISTIC: y[n_obs] in {0,1}                                               */
    double scalar0;      /* MVGAUSS: sum(log diag L) (constant of the log-density)                    */
    const double* m1;    /* MVGAUSS: L^-T [n][n] row-major (p0 = solve_triangular(L^T, z) = L^-T z)   */
    const double* m2;    /* MVGAUSS: Cholesky factor L [n][n] row-major (v0 = Sigma p0 = L z)         */
    const b200_ir* ir;   /* IR: the model as data (see above)                                         */
} b200_model_desc;

/* NumPy PCG64 stream state (numpy.random.PCG64().state["state"]): 128-bit LCG state and increment.
 * One `step` stream per chain (tree direction / multinomial picks, reference order: SURVEY 8a a15). */
typedef struct b200_pcg64 {
    uint64_t state_hi, state_lo;
    uint64_t inc_hi, inc_lo;
} b200_pcg64;

/* Per-chain sampler state between calls: what BaseHMC.sampling_state carries for a NUTS/HMC chain with a diagonal adaptive
 * potential (hmc/base_hmc.py:61-71: iter_count, step_adapt, potential; step_sizes.py:26-38 StepSizeState;
 * quadpotential.py:189-208 QuadPotentialDiagAdaptState with its two WeightedVarianceState, :396-403).  Arrays of length C
 * ([C][n] where noted) in the memory space of the call.  Used (i) to checkpoint / resume chains, (ii) to run warm-up in
 * windows with the estimators pooled over chains and GPUs in between (pymc_b200.parallel.pooled_warmup).
 * For DIAG_ADAPT_GRAD the four estimator arrays hold (mean, var) of the draws (fg_*) and of the gradients (bg_*). */
typedef struct b200_chain_state {
    double* q;          /* [C][n] current position                                              */
    double* log_step;   /* DualAverageAdaptation._log_step                                        */
    double* log_bar;    /*                       ._log_bar                                         */
    double* hbar;       /*                       ._hbar                                            */
    int32_t* da_count;  /*                       ._count                                           */
    int32_t* n_samples; /* QuadPotentialDiagAdapt._n_samples                                      */
    int32_t* window;    /*                       .adaptation_window                               */
    double* var;        /* [C][n]                ._var                                             */
    double* fg_n;       /* foreground estimator: n_samples, mean [C][n], raw_var [C][n]            */
    double* fg_mean;
    double* fg_m2;
    double* bg_n;       /* background estimator                                                    */
    double* bg_mean;
    double* bg_m2;
    int64_t* n_grad;    /* logp+grad evaluations so far                                            */
} b200_chain_state;

/* Sampler configuration: the keyword surface of pm.NUTS / BaseHMC (hmc/nuts.py:132, hmc/base_hmc.py:82-98). */
typedef struct b200_nuts_cfg {
    int32_t chains;              /* C: independent chains in this call                                */
    int32_t tune;                /* warm-up iterations (adaptation on)                                */
    int32_t draws;               /* iterations after stop_tuning()                                    */
    int32_t max_treedepth;       /* default 10                                                        */
    int32_t early_max_treedepth; /* default 8: used while tuning and iter_count < 200                 */
    int32_t adapt_step_size;     /* default 1                                                         */
    int32_t mass_kind;           /* B200_MASS_*                                                       */
    int32_t momentum_source;     /* B200_MOMENTUM_*                                                   */
    int32_t store_warmup;        /* 1: outputs hold tune+draws iterations; 0: only the `draws` part   */
    int32_t chain_offset;        /* global index of chain 0 of this call (multi-GPU shards): keys the Philox stream */
    double step_scale;           /* default 0.25; eps0 = step_scale / n**0.25 (base_hmc.py:161)       */
    double target_accept;        /* default 0.8                                                       */
    double gamma;                /* default 0.05                                                      */
    double k;                    /* default 0.75                                                      */
    double t0;                   /* default 10                                                        */
    double Emax;                 /* default 1000                                                      */
    /* QuadPotentialDiagAdapt parameters (quadpotential.py:216-229; init_nuts uses weight 10) */
    double mass_initial_weight;  /* default 10                                                        */
    int32_t adaptation_window;   /* default 101                                                       */
    int32_t discard_window;      /* default 50                                                        */
    uint64_t philox_seed;        /* key for B200_MOMENTUM_DEVICE_PHILOX                               */
    int32_t sampler;             /* B200_SAMPLER_*; default NUTS                                      */
    int32_t max_steps;           /* HMC: default 1024                                                 */
    double path_length;          /* HMC: default 2.0                                                  */
    double mass_alpha;           /* DIAG_ADAPT_GRAD: decay rate, default 0.02                         */
    int32_t stop_adaptation;     /* DIAG_ADAPT_GRAD: stop after this many updates; < 0 = never (init_nuts: tune - 50 if tune > 250) */
    int32_t iter_begin;          /* this call runs iterations [iter_begin, iter_begin + iter_count) of the tune + draws schedule */
    int32_t iter_count;          /* 0 = all remaining (tune + draws - iter_begin); outputs / z hold exactly these iterations   */
    const b200_chain_state* resume;  /* NULL: chains start fresh (iter_begin must be 0); else the state exported by the previous call */
    b200_chain_state* save;          /* NULL or where to export the state after the last iteration of this call                */
    int32_t constrain_draws;     /* 1: draws_out holds the CONSTRAINED values (backward transforms of b200_model_set_transforms
                                  * applied where a draw is recorded: the per-draw post-processing of backends/ndarray.py:108
                                  * fused into the kernel); 0: unconstrained positions */
    int32_t mass_update_window;  /* DENSE_ADAPT: covariance + Cholesky refresh every this many tuning draws; 0 = default 1     */
    double adaptation_window_multiplier; /* DENSE_ADAPT: window growth factor at every switch; 0 = default 2 (quadpotential.py:758) */
} b200_nuts_cfg;

/* Per-draw sampler statistics, struct-of-arrays [C][T] with T = store_warmup ? tune+draws : draws.
 * Names follow NUTS.stats_dtypes_shapes (hmc/nuts.py:110-130).  Any pointer may be NULL (not recorded).
 * All pointers live in the memory space given by `mem`. */
typedef struct b200_stats {
    int32_t* depth;
    int32_t* tree_size;            /* == n_proposals == leapfrog gradient evaluations of the draw     */
    int32_t* index_in_trajectory;
    uint8_t* diverging;
    uint8_t* reached_max_treedepth;
    double* step_size;
    double* step_size_bar;
    double* mean_tree_accept;
    double* energy;
    double* energy_error;
    double* max_energy_error;
    double* model_logp;
} b200_stats;

/* Per-chain end-of-run state, arrays of length C (any pointer may be NULL). */
typedef struct b200_chain_summary {
    int64_t* grad_evals;     /* total logp+grad evaluations incl. the one at the start of every draw  */
    int32_t* bad_energy_at;  /* -1, or the iteration at which "Bad initial energy" froze the chain    */
    double* final_step_size; /* exp(log_bar) after tuning                                            */
    double* final_var;       /* [C][n] diagonal inverse-mass ("_var") at the end of the run           */
    double* final_cov;       /* [C][n][n] DENSE_ADAPT: the chain's covariance ("_cov") at the end of the run */
} b200_chain_summary;

int b200_version(void);
const char* b200_last_error(void);
/* sizeof() of the ABI structs as this library was compiled, so a host binding can verify its mirrors before passing
 * pointers: which = 0 b200_model_desc, 1 b200_nuts_cfg, 2 b200_stats, 3 b200_chain_summary, 4 b200_pcg64, 5 b200_ir,
 * 6 b200_ir_var, 7 b200_ir_prior, 8 b200_ir_term, 9 b200_ir_lik, 10 b200_ir_ar1, 11 b200_ir_param, 12 b200_ir_factor,
 * 13 b200_chain_state;
 * -1 for an unknown index. */
int b200_struct_size(int which);

/* Number of visible CUDA devices (0 if none / no driver): lets a host binding fail loudly. */
int b200_device_count(void);
/* Binds the calling thread to a device (cudaSetDevice).  One process per GPU. */
int b200_set_device(int device);

/* Replaces: Model.logp_dlogp_function(ravel_inputs=True) -> ValueGradFunction
 *           (pymc/model/core.py:464-529, :142-305) -- the compile step. */
int b200_model_create(const b200_model_desc* desc, b200_model** out);
/* Arithmetic of the dense contractions of a GEMM-shaped model (affects b200_logp_dlogp and b200_nuts_run of that handle).
 *   B200_PRECISION_FP64      IEEE fp64 on the fp64 tensor path (DMMA) -- the parity mode, default.
 *   B200_PRECISION_TC_FP16X2 LOGISTIC and MVGAUSS: the dense contractions on the fp16 tensor cores (wgmma, TMA) with
 *                            every fp64 operand split into two fp16 pieces and fp32 accumulation, drained into fp64 every
 *                            256 rows (logistic) / into compensated sums every 64 terms (GEMM); operands are scaled by
 *                            exact powers of two per row / column first, so at any data scale every output is within
 *                            2^-18 S of the exact value, S = the sum of |terms| it is made of (tests/test_gpu_contractions.py;
 *                            gradient within 1e-6 of its largest entry at unit-scale data, tests/test_gpu_tc.py).
 * The reference computes in floatX = float64 (pymc/pytensorf.py); this is the "tensor cores where the logp really is a
 * dense matvec" performance mode of north_star, with its error stated next to the number. */
#define B200_PRECISION_FP64 0
#define B200_PRECISION_TC_FP16X2 1
int b200_model_set_precision(b200_model* model, int32_t mode);
void b200_model_destroy(b200_model* model);
/* Per-element backward transforms of the value variables (kind[n]: 0 identity, 1 exp, 2 lo + (hi - lo) sigmoid), used when
 * b200_nuts_cfg.constrain_draws is set.  Replaces the compiled "unobserved values" function the reference evaluates per
 * draw (pymc/backends/base.py:184-191, ndarray.py:108; transforms pymc/logprob/transforms.py:880-891, :1026-1045). */
int b200_model_set_transforms(b200_model* model, const int8_t* kind, const double* lo, const double* hi);
/* Fixed dense mass matrix for B200_MASS_DENSE runs of ANY model (host matrices [n][n] row-major, copied):
 *   velocity v = cov . p,  momentum p0 = mp0 . z,  its velocity v0 = mv0 . z   with z ~ N(0, I).
 * QuadPotentialFull(cov)   (quadpotential.py:680-725): mp0 = L^-T, mv0 = L with L = cholesky(cov, lower)
 * QuadPotentialFullInv(A)  (quadpotential.py:633-677): cov = A^-1, mp0 = cholesky(A, lower), mv0 = mp0^-T
 * (the host binding computes the factors; see pymc_b200.engine.CompiledModel.set_dense_mass).  Dense-mass runs advance all
 * chains in lock step: one model evaluation kernel + one fp64 tensor-core GEMM (Sigma . grad) per leapfrog. */
int b200_model_set_dense_mass(b200_model* model, const double* cov, const double* mp0, const double* mv0);
int b200_model_n(const b200_model* model);

/* Replaces: ValueGradFunction._pytensor_function(q) -> (logp, dlogp), batched over C points
 *           (built pymc/model/core.py:232-267; called hmc/integration.py:51-52,70,129).
 * q[C][n] row-major, logp[C], grad[C][n]; `mem` is B200_MEM_HOST or B200_MEM_DEVICE for all three. */
int b200_logp_dlogp(b200_model* model, const double* q, int32_t C, double* logp, double* grad,
                    int32_t mem, void* stream);

/* Replaces: CpuLeapfrogIntegrator.compute_state + n_steps x CpuLeapfrogIntegrator._step with a
 *           diagonal potential (hmc/integration.py:68-75, :109-145; quadpotential.py:610-630).
 * In/out (struct-of-arrays, one row per chain): q,p,v,grad [C][n]; energy, logp [C]; idx [C].
 * var[C][n] is the diagonal inverse mass, eps[C] the signed step size.  If n_steps == 0 only the
 * start state (grad, v, energy, logp) is computed from (q, p). */
int b200_leapfrog(b200_model* model, const double* var, const double* eps, int32_t n_steps,
                  int32_t C, double* q, double* p, double* v, double* grad, double* energy,
                  double* logp, int64_t* idx, int32_t mem, void* stream);

/* Replaces the whole multi-chain sampling loop for NUTS:
 *   _sample_many/_mp_sample/_iter_sample   pymc/sampling/mcmc.py:1385-1583   (chains x iterations)
 *   BaseHMC.astep                          hmc/base_hmc.py:196-288           (one draw)
 *   NUTS._hamiltonian_step / _Tree         hmc/nuts.py:204-489               (tree doubling, U-turn, picks)
 *   CpuLeapfrogIntegrator                  hmc/integration.py:68-145         (leapfrog)
 *   QuadPotentialDiag(Adapt)               hmc/quadpotential.py:211-355,582-630
 *   DualAverageAdaptation                  pymc/step_methods/step_sizes.py:41-84
 * All chains run inside one persistent kernel; there is no host round-trip per leapfrog or per draw.
 *
 *   q0[C][n]          start points (unconstrained)
 *   var0[C][n]        initial diagonal inverse mass (ones for jitter+adapt_diag); NULL = ones
 *   mean0[C][n]       DIAG_ADAPT: initial mean of the foreground estimator (init_nuts passes the mean
 *                     start point over chains, mcmc.py:1890); NULL = zeros
 *   eps0[C]           optional per-chain initial step size overriding step_scale / n**0.25 (a chain resumed
 *                     from a saved sampling_state carries its own step size, base_hmc.py:61-71); NULL = default
 *   rng[C]            per-chain NumPy PCG64 `step` stream states; updated in place on return
 *   z[C][Ttot][n]     momentum noise when momentum_source == B200_MOMENTUM_HOST_BUFFER, else NULL
 *   draws_out[C][T][n]  accepted positions (unconstrained), T per `store_warmup`
 *   stats, summary    see above; their pointers are in the same memory space
 *   mem               memory space of ALL the buffers above
 */
int b200_nuts_run(b200_model* model, const b200_nuts_cfg* cfg, const double* q0, const double* var0,
                  const double* mean0, const double* eps0, b200_pcg64* rng, const double* z, double* draws_out,
                  const b200_stats* stats, const b200_chain_summary* summary, int32_t mem,
                  void* stream);

/* Pointwise log-likelihood of likelihood factor `lik` of an IR model for D unconstrained draws:
 * out[d][i] = log p(y_i | draws[d]).  Replaces pm.compute_log_likelihood's per-draw compiled function
 * (pymc/stats/log_density.py:31-77, :129-195): the `log_likelihood` group of the InferenceData. */
int b200_pointwise_loglik(b200_model* model, int32_t lik, const double* draws /*[D][n]*/, int64_t D,
                          double* out /*[D][N]*/, int32_t mem, void* stream);

/* Device time (ms, CUDA events on the launching stream) and launch count of the kernels of the
 * most recent b200_nuts_run / b200_logp_dlogp / b200_leapfrog call on this thread. */
int b200_last_kernel_ms(double* ms, int32_t* launches);

/* fp64 FMA micro-benchmark: sustained DFMA throughput in TFLOP/s of this device (roofline
 * denominator for compute-bound configs; MEASURED_PEAKS.json has only HBM and bf16). */
int b200_measure_fp64_tflops(double* tflops);
/* The same for the fp64 tensor path (mma.sync m8n8k4.f64, SASS DMMA.8x8x4) that the GEMM-shaped models
 * (LOGISTIC, MVGAUSS) contract on. */
int b200_measure_dmma_tflops(double* tflops);

#ifdef __cplusplus
}
#endif
#endif /* B200NUTS_H */
