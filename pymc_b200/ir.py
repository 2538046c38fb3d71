"""ModelSpec IR: what a PyMC model looks like to the sampling engine (SURVEY.md section 7 "Hard parts", 8b, 8f-2).

In the reference the sampler sees a model as ONE compiled callable ``q -> (logp, dlogp)`` over the raveled, transformed
value variables (``Model.logp_dlogp_function``, pymc/model/core.py:464-529; summation of factors :688-690; transforms and
their Jacobians pymc/logprob/transforms.py:880-891, :1026-1073).  The IR keeps exactly that structure in data:

    value variables   ordered, each with a size and a transform (None | "log" | "interval"(lo, hi))
    factors           a closed set, each contributing logp(x) where x are the CONSTRAINED values
        Prior         elementwise density of one variable; parameters are constants or scalar variables (hierarchies);
                      a Normal / StudentT location may be a Linear predictor (group-level predictors, nested groups)
        Likelihood    observed y_i with a linear predictor  eta_i = sum_t coef_t[i] * prod_f x_f[idx_f[i]]
                      (affine / indexed / bilinear links: intercepts, slopes x data, group effects, scale * offset ...)
        AR1           h_0 ~ Normal(0, init_sigma), h_t - phi h_{t-1} ~ Normal(0, sigma)   (phi = 1: Gaussian random walk)

``lower()`` flattens a model into the arrays of the C ABI's ``b200_ir`` (include/b200nuts.h); the engine evaluates it with
ONE generic fused logp+gradient device function (csrc/ir_model.cuh) inside the same persistent NUTS kernel -- a new model
needs no new CUDA.  Models whose IR matches a hand-specialised kernel (Eight Schools, Radon) are routed to it by
``specialise()``: the enum kinds of round 1 are fast paths behind the IR, not the interface.

``oracle/ir_numpy.py`` evaluates the same IR in NumPy (test infrastructure).
"""
from __future__ import annotations

import copy
import dataclasses
from dataclasses import dataclass, field

import numpy as np

# ids shared with include/b200nuts.h ------------------------------------------------------------------------------------
TRANSFORMS = {None: 0, "log": 1, "interval": 2,
              "ordered": 3, "ordered_positive": 4,  # Ordered() / Ordered(positive=True), transforms.py:79-120
              "simplex": 5}  # SimplexTransform, transforms.py:1091-1116: Var.size is K - 1, the constrained value K weights
ORDERED_TRANSFORMS = ("ordered", "ordered_positive")
# An ordered variable is not constrained elementwise (a cumulative sum): it takes only real-line priors, and
# ordered_positive also counts as positive support (csrc/b200nuts.cu: prepare_ir, same words)
REAL_LINE_PRIORS = ("flat", "normal", "studentt", "cauchy")
ORDERED_PRIOR = ("an ordered variable takes only real-line priors (flat, normal, studentt, cauchy, or a latent normal / "
                 "studentt); ordered_positive also admits the positive priors")
# priors: name -> (id, number of parameters)
PRIOR_DISTS = {
    "flat": (0, 0),          # Flat / HalfFlat: logp 0                                  continuous.py:364-383, :400-419
    "normal": (1, 2),        # (mu, sigma)                                              continuous.py:526-527
    "halfnormal": (2, 1),    # (sigma)                                                  continuous.py:909-911
    "cauchy": (3, 2),        # (alpha, beta)                                            continuous.py:2287-2288
    "halfcauchy": (4, 1),    # (beta)                                                   continuous.py:2383-2385
    "exponential": (5, 1),   # (lam); PyMC's logp is written in mu = 1/lam              continuous.py:1478-1480
    "studentt": (6, 3),      # (nu, mu, sigma); nu constant                             continuous.py:1936-1944
    "uniform": (7, 2),       # (lower, upper) constants                                 continuous.py:309-314
    "gamma": (8, 2),         # (alpha, beta) constants                                  continuous.py:2512-2515
    "beta": (9, 2),          # (alpha, beta) constants                                  continuous.py:1250-1256
    "lognormal": (10, 2),    # (mu, sigma)                                              continuous.py:1807-1814
    "dirichlet": (11, 1),    # (a): K constants > 0 or one broadcast; on a simplex only  multivariate.py:557-585
    "inversegamma": (12, 2), # (alpha, beta) constants                                  continuous.py:2631-2640
}
# likelihoods: name -> id
LIK_DISTS = {
    "normal": 0,             # y_i ~ Normal(eta_i, sigma)                               continuous.py:526-527
    "bernoulli_logit": 1,    # y_i ~ Bernoulli(logit_p = eta_i)                         discrete.py:362-367 (stabilised forms)
    "poisson_log": 2,        # y_i ~ Poisson(mu = exp(eta_i))                           discrete.py:581-586
    "studentt": 3,           # y_i ~ StudentT(nu, eta_i, sigma)                         continuous.py:1936-1944
    "normal_logvar": 4,      # y_i ~ Normal(0, exp(eta_i / 2))   (stochastic volatility observation)
    "binomial_logit": 5,     # y_i ~ Binomial(trials, logit_p = eta_i)                  discrete.py:141-152 (stabilised forms)
    "negative_binomial_log": 6,  # y_i ~ NegativeBinomial(mu = exp(eta_i), alpha)       discrete.py:700-745
    "gamma_log": 7,          # y_i ~ Gamma(alpha, beta = alpha exp(-eta_i))             continuous.py:2478-2521
    "censored_normal": 8,    # y_i ~ Censored(Normal(eta_i, sigma), lower, upper)       logprob/censoring.py:213-248
    "truncated_normal": 9,   # y_i ~ TruncatedNormal(eta_i, sigma, lower, upper)        continuous.py:720-747
    "ordered_logistic": 10,  # y_i ~ OrderedLogistic(eta_i, cutpoints)                  discrete.py:1231-1326, :1190-1206
    "ordered_probit": 11,    # y_i ~ OrderedProbit(eta_i, cutpoints, sigma)             discrete.py:1329-1432, :1190-1206
    "zero_inflated_poisson": 12,            # ZeroInflatedPoisson(psi, mu = exp(eta_i))            mixture.py:577-638
    "zero_inflated_binomial": 13,           # ZeroInflatedBinomial(psi, trials, logit_p = eta_i)   mixture.py:641-702
    "zero_inflated_negative_binomial": 14,  # ZeroInflatedNegativeBinomial(psi, exp(eta_i), alpha) mixture.py:705-802
    "hurdle_poisson": 15,                   # HurdlePoisson(psi, mu = exp(eta_i))                  mixture.py:873-922
    "hurdle_negative_binomial": 16,         # HurdleNegativeBinomial(psi, exp(eta_i), alpha)       mixture.py:925-978
    "hurdle_gamma": 17,                     # HurdleGamma(psi, alpha, beta = alpha / exp(eta_i))   mixture.py:981-1034
    "weibull_log": 18,             # y_i ~ Weibull(alpha, beta = exp(eta_i)); Exponential(scale = exp(eta_i)): alpha = 1
    "lognormal": 19,               # y_i ~ LogNormal(mu = eta_i, sigma)                          continuous.py:1723-1846
    "censored_weibull_log": 20,    # y_i ~ Censored(Weibull(alpha, exp(eta_i)), lower, upper)     continuous.py:2740-2831
    "censored_lognormal": 21,      # y_i ~ Censored(LogNormal(eta_i, sigma), lower, upper)
    "truncated_weibull_log": 22,   # y_i ~ Truncated(Weibull(alpha, exp(eta_i)), lower, upper)
    "truncated_lognormal": 23,     # y_i ~ Truncated(LogNormal(eta_i, sigma), lower, upper)
    "normal_mixture": 24,    # y_i ~ NormalMixture(w, eta_i + mu_k, sigma_k)                mixture.py:469-494, :529-546
    "poisson_mixture": 25,   # y_i ~ Mixture(w, Poisson(lam_k exp(eta_i)))
    "beta_logit": 26,            # y_i ~ Beta(mu = sigmoid(eta_i), nu = phi)               continuous.py:1131-1262, :1238-1240
    "beta_binomial_logit": 27,   # y_i ~ BetaBinomial(n_i, phi mu_i, phi (1 - mu_i))       discrete.py:178-262
}
# Zero-inflated and hurdle observations: ``Likelihood.psi`` is the probability of the count / positive component, a
# constant in (0, 1), a Ref to a scalar variable with an interval transform inside [0, 1], or a Linear: the logit of psi.
# Each is its family (ZI_FAMILY) with the family's parameter slot (trials, alpha).  Lowered with the psi block one past the
# predictor's terms and nu = 0 (psi itself) or the number of terms of logit(psi) (include/b200nuts.h).
ZI_FAMILY = {"zero_inflated_poisson": "poisson_log", "zero_inflated_binomial": "binomial_logit",
             "zero_inflated_negative_binomial": "negative_binomial_log", "hurdle_poisson": "poisson_log",
             "hurdle_negative_binomial": "negative_binomial_log", "hurdle_gamma": "gamma_log"}
ZI_LIKS = tuple(ZI_FAMILY)
# the refusals (csrc/b200nuts.cu: prepare_ir, same words)
PSI_NU = "nu must be an integer >= 0: 0 for psi itself, m >= 1 for the m terms of logit(psi)"
PSI_BLOCK = ("the psi block is one constant or one unindexed scalar variable (nu = 0), or the terms of logit(psi) "
             "(nu >= 1)")
PSI_CONST = "a constant psi must be finite and lie in (0, 1)"
PSI_ONE = ("psi = 1 leaves no zero component: write the plain likelihood (poisson_log, binomial_logit, "
           "negative_binomial_log or gamma_log)")
PSI_VAR = "a psi variable must be scalar with an interval transform inside [0, 1] (0 <= lo < hi <= 1)"
ZI_Y = "y must be integers >= 0"
ZIB_Y = "y must be integers with 0 <= y <= trials"
HG_Y = "y must be finite and >= 0"
ZIP_SLOT = "zero_inflated_poisson and hurdle_poisson take no sigma, trials or alpha"
# Ordinal observations: y_i in 0..K-1 and ``Likelihood.cutpoints``, a Ref to a variable of size K - 1 (ordered unless
# K = 2) or K - 1 constants, finite and strictly increasing; lowered with nu = K and the cutpoint term one past the
# predictor's terms (include/b200nuts.h)
ORDINAL_LIKS = ("ordered_logistic", "ordered_probit")
ORD_K = "an ordinal likelihood needs K >= 2 categories"
ORD_Y = "y must be integers in [0, K - 1]"
CUT_SIZE = "the cutpoint variable must have size K - 1"
CUT_ORDERED = "a cutpoint variable of size > 1 needs an ordered transform"
CUT_CONST = "constant cutpoints must be finite and strictly increasing"
LOGISTIC_SIGMA = "ordered_logistic has no sigma"
# Normal observations with bounds: ``Likelihood.lower`` / ``.upper`` (None, a constant or one value per observation, -inf /
# +inf where that side is open); lowered as the [3][N] block (y, lower, upper) of include/b200nuts.h
BOUNDED_LIKS = ("censored_normal", "truncated_normal")
# Survival (time-to-event) observations y_i > 0 with a log link: the Weibull (the Exponential is its alpha = 1) and the
# LogNormal, plain, censored or truncated.  Bounds as for the Normal ones (``Likelihood.lower`` / ``.upper``, lowered as the
# [3][N] block), where a lower bound of 0 or -inf is an open side; the Weibull's shape is ``Likelihood.alpha``, the
# LogNormal's scale ``Likelihood.sigma`` (include/b200nuts.h)
WEIBULL_LIKS = ("weibull_log", "censored_weibull_log", "truncated_weibull_log")
LOGNORMAL_LIKS = ("lognormal", "censored_lognormal", "truncated_lognormal")
SURVIVAL_LIKS = WEIBULL_LIKS + LOGNORMAL_LIKS
SURVIVAL_BOUNDED = ("censored_weibull_log", "censored_lognormal", "truncated_weibull_log", "truncated_lognormal")
SIGMA_LIKS = ("normal", "studentt") + BOUNDED_LIKS + ("ordered_probit",) + LOGNORMAL_LIKS  # parameter slot: sigma
# the support rule of bounded observations (csrc/b200nuts.cu: prepare_ir, same words)
BOUND_SIDES = "lower must not be +inf or NaN and upper must not be -inf or NaN"
BOUND_ORDER = "lower < upper must hold for every observation"
BOUND_Y = "y must be finite and lie in [lower, upper] for every observation"
TRUNC_OPEN = "truncated_normal needs a finite lower or upper bound; with neither side bounded, write the likelihood as normal"
# the support rule of survival observations (csrc/b200nuts.cu: prepare_ir, same words)
SURV_Y = "y must be finite and > 0 for every observation"
SURV_SIDES = "lower must be finite and >= 0 or -inf (0 and -inf: open) and upper > 0 or +inf (open), neither NaN"
SURV_TRUNC_OPEN = ("a truncated survival likelihood needs a finite lower bound > 0 or a finite upper bound; with neither, "
                   "write the plain likelihood")
SURV_PLAIN = "lower / upper belong to the censored_ and truncated_ forms"
WEIBULL_SIGMA = "a Weibull likelihood has no sigma (its parameter is alpha)"
DISPERSION_LIKS = ("negative_binomial_log", "gamma_log")  # their `alpha` is a constant or a Ref
# Finite mixtures of K >= 2 components, log p(y_i) = logsumexp_k(log w_k + log f_k(y_i)): ``Likelihood.weights`` (a Ref to a
# simplex variable or K constants) and ``.components`` (mu_k / lam_k: a Ref to a variable of size K or K constants); the
# Normal's ``sigma`` is one or K constants or a Ref to a variable of size 1 or K.  The predictor's terms may be empty.
# Lowered with nu = K and the weights, component and sigma blocks one past the predictor's terms (include/b200nuts.h).
MIXTURE_LIKS = ("normal_mixture", "poisson_mixture")
# the rules of simplex variables, Dirichlet priors and mixtures (csrc/b200nuts.cu: prepare_ir, same words)
SIMPLEX_USE = "a simplex variable may be used only as a mixture's weights"
SIMPLEX_PRIOR = "a simplex variable carries exactly one prior, a dirichlet of length K = size + 1"
DIRICHLET_VAR = "a dirichlet prior is only allowed on a simplex variable"
DIRICHLET_A = "a dirichlet's a must be one finite constant > 0 (K equal constants lower to it)"
MIX_K = "a mixture needs K >= 2 components; with K = 1, write the plain likelihood (normal or poisson_log)"
MIX_Y_NORMAL = "y must be finite"
MIX_WEIGHTS = "the weights must be a simplex variable of size K - 1 or K finite constants >= 0 that sum to 1"
MIX_MU = "mu must be a variable of size K with no transform or an ordered one, or K finite constants"
MIX_LAM = ("lam must be a variable of size K with positive support (log, ordered_positive, or an interval with lo >= 0), "
           "or K finite constants > 0")
MIX_SIGMA = "sigma must be a finite constant > 0, K of them, or a variable of size 1 or K with positive support"
MIX_SLOTS = "a mixture takes no alpha, trials, lower / upper, cutpoints or psi, and poisson_mixture no sigma"
# Beta regression with a logit mean, mu_i = sigmoid(eta_i), and a precision ``Likelihood.phi`` (PyMC's ``nu`` of
# ``Beta(mu, nu)``): a finite constant > 0 or a Ref to a scalar variable with positive support.  beta_logit observes
# y_i in (0, 1); beta_binomial_logit observes counts y_i of ``Likelihood.trials`` (one constant or one per observation),
# with a = phi mu_i and b = phi (1 - mu_i).  Lowered with phi in the parameter slot and, for the BetaBinomial, the
# [2][N] block (y, trials) (include/b200nuts.h).
BETA_LIKS = ("beta_logit", "beta_binomial_logit")
# the support rule of Beta / BetaBinomial observations (csrc/b200nuts.cu: prepare_ir, same words)
BETA_Y = ("y must be finite with 0 < y < 1 for every observation (0 and 1 are outside the Beta's support; a "
          "zero/one-inflated Beta is not provided)")
BB_TRIALS = "trials must be finite integers >= 0"
BETA_SLOTS = ("beta_logit and beta_binomial_logit take phi, and no sigma, alpha, cutpoints, psi, weights, components or "
              "lower / upper")
BETA_TRIALS = "trials belong to beta_binomial_logit (a Beta observes proportions, not counts)"
# Spectral terms: a Hilbert-space approximate GP (pm.gp.HSGP, non-centred, hsgp_approx.py:453-473) as a design term whose
# column weights depend on hyperparameters, f = Phi (z * s(theta)) with s_k = amplitude sqrt(S(omega_k; ls)) and S the
# power spectral density of ``cov`` (cov.py:574-583, :690-710, :743-761).  Lowered as the ABI's spectral term
# (include/b200nuts.h), or as a plain design term when ls and amplitude are constants.
COV_FUNCS = {"expquad": 1, "matern52": 2, "matern32": 3}
# the rules of spectral terms (csrc/b200nuts.cu: prepare_ir, same words)
SPEC_PHI = "a spectral term's Phi must be finite with shape (N, M), M the size of its variable"
SPEC_Z = "a spectral term's variable must be one whole variable with no index and no transform"
SPEC_OMEGA = "omega must have shape (M, D), D >= 1, with finite entries >= 0"
SPEC_COV = "cov must be expquad, matern52 or matern32"
SPEC_LS = "ls must be a finite constant > 0, D of them, or a variable of size 1 or D with positive support"
SPEC_AMP = "amplitude must be a finite constant > 0 or a scalar variable with positive support"
# The support rule.  The device evaluates a density's formula wherever it is asked to, so every variable must be kept
# inside its prior's support by its transform, and every scale parameter must be positive:
POSITIVE_PRIORS = ("halfnormal", "halfcauchy", "exponential", "gamma", "lognormal", "inversegamma")  # a log transform, or interval lo >= 0
SCALE_PARAMS = {"normal": {1: "sigma"}, "lognormal": {1: "sigma"}, "halfnormal": {0: "sigma"}, "cauchy": {1: "beta"},
                "halfcauchy": {0: "beta"}, "exponential": {0: "lam"}, "studentt": {2: "sigma"}}
POSITIVE_SUPPORT = "a scalar variable with positive support (a log transform, or an interval with lo >= 0)"
NEGBIN_POISSON_ALPHA = 1e10  # above: the NegativeBinomial density is its Poisson(mu) limit (discrete.py:727-735)
SIGMA_NONE, SIGMA_CONST, SIGMA_REF, SIGMA_OBS = 0, 1, 2, 3
MAX_TERM_FACTORS = 3
# priors whose location may be a Linear predictor: name -> (location slot, scale slot).  Such a prior is lowered to a
# latent factor (see ``lower``), which also takes one constant scale per element.
LINEAR_PRIORS = {"normal": (0, 1), "studentt": (1, 2)}


def _positive_support(v) -> bool:
    return v.transform in ("log", "ordered_positive") or (v.transform == "interval" and v.bounds[0] >= 0.0)


def ordered_backward(z: np.ndarray, positive: bool) -> np.ndarray:
    """Ordered.backward (transforms.py:96-106) along the last axis: x_0 = z_0 (positive: exp z_0), x_k = x_{k-1} + exp z_k,
    summed in np.cumsum's order (k ascending), as the device does."""
    d = np.exp(z)
    if not positive:
        d[..., 0] = z[..., 0]
    return np.cumsum(d, axis=-1)


def simplex_backward(z: np.ndarray) -> np.ndarray:
    """SimplexTransform.backward (transforms.py:1101-1105) along the last axis: w = softmax([z, -sum z])."""
    z = np.asarray(z, dtype=np.float64)
    ze = np.concatenate([z, -np.sum(z, axis=-1, keepdims=True)], axis=-1)
    e = np.exp(ze - np.max(ze, axis=-1, keepdims=True))
    return e / np.sum(e, axis=-1, keepdims=True)


def spectral_log_const(cov: str, D: int) -> tuple[float, float, float]:
    """(log C_D, nu, c) of S = C_D prod_d l_d exp(h(Q)) with h = -Q / 2 (expquad, nu = 0) or -nu log(c + Q) (Matern)."""
    from scipy.special import gammaln

    if cov == "expquad":
        return 0.5 * D * np.log(2.0 * np.pi), 0.0, 0.0
    order, den = (2.5, 0.75) if cov == "matern52" else (1.5, 0.5)
    nu, c = 0.5 * D + order, 2.0 * order
    return D * np.log(2.0) + 0.5 * D * np.log(np.pi) + gammaln(nu) + order * np.log(c) - np.log(den * np.sqrt(np.pi)), nu, c


def spectral_log_scale(cov: str, omega, ls, amplitude) -> np.ndarray:
    """log s_k = log amplitude + (log C_D + sum_d log l_d + h(Q_k)) / 2 with Q_k = sum_d l_d^2 omega_kd^2, as [..., M] for
    ls [..., D] and amplitude [...] (leading axes: draws)."""
    omega = np.asarray(omega, dtype=np.float64)
    ls = np.asarray(ls, dtype=np.float64)
    log_c, nu, c = spectral_log_const(cov, omega.shape[1])
    Q = np.einsum("...d,kd->...k", ls * ls, omega * omega)
    h = -0.5 * Q if cov == "expquad" else -nu * np.log(c + Q)
    base = np.log(np.asarray(amplitude, dtype=np.float64)) + 0.5 * (log_c + np.sum(np.log(ls), axis=-1))
    return base[..., None] + 0.5 * h


def hsgp_basis(X, m, c=None, L=None, drop_first: bool = False):
    """(Phi [N][M], omega [M][D], centre [D], L [D]) of the Hilbert-space approximation with m[d] basis functions per
    dimension, by the method of pm.gp.HSGP.prior_linearized: the inputs are centred at (max + min) / 2; the half-width L_d
    is c (max - min) / 2 unless L is given; the eigenvalues of the Laplacian on [-L, L]^D are lambda_jd = (pi j_d / (2
    L_d))^2 for j_d = 1..m[d], combined over the dimensions in np.meshgrid's order; omega = sqrt(lambda) and phi_j(x) =
    prod_d L_d^(-1/2) sin(sqrt(lambda_jd) (x_d + L_d)).  ``drop_first`` drops the first basis function."""
    X = np.asarray(X, dtype=np.float64)
    X = X[:, None] if X.ndim == 1 else X
    D = X.shape[1]
    m = [int(m)] * D if np.ndim(m) == 0 else [int(v) for v in m]
    centre = 0.5 * (X.max(axis=0) + X.min(axis=0))
    Xs = X - centre
    if L is None:
        if c is None:
            raise ValueError("hsgp_basis needs c or L")
        L = np.asarray(c, dtype=np.float64) * 0.5 * (X.max(axis=0) - X.min(axis=0))
    L = np.broadcast_to(np.asarray(L, dtype=np.float64), (D,)).copy()
    grid = np.meshgrid(*[np.arange(1, 1 + md) for md in m])
    J = np.stack([g.ravel() for g in grid], axis=1).astype(np.float64)  # [M][D]
    omega = np.pi * J / (2.0 * L)
    Phi = np.ones((X.shape[0], J.shape[0]))
    for d in range(D):
        Phi *= np.sin(omega[:, d][None, :] * (Xs[:, d][:, None] + L[d])) / np.sqrt(L[d])
    i = int(bool(drop_first))
    return Phi[:, i:], omega[i:], centre, L


def spectral_weights(ir, t, x: dict) -> np.ndarray:
    """s(theta) [..., M] of spectral term t at the constrained values ``x`` (rv name -> draws, as ``constrain`` returns)."""
    sp = t.spectral
    D = np.shape(sp.omega)[1]
    if isinstance(sp.ls, Ref):
        v = ir.var(sp.ls.var)
        ls = np.asarray(x[v.rv_name], dtype=np.float64)
        ls = ls[..., None] if v.size == 1 else ls  # an isotropic lengthscale (or D = 1)
    else:
        ls = np.asarray(sp.ls, dtype=np.float64).reshape(-1)
    amp = np.asarray(x[ir.var(sp.amplitude.var).rv_name] if isinstance(sp.amplitude, Ref) else sp.amplitude,
                     dtype=np.float64)
    lead = np.broadcast_shapes(ls.shape[:-1], amp.shape)
    ls = np.broadcast_to(ls, lead + (D,))
    return np.exp(spectral_log_scale(sp.cov, sp.omega, ls, np.broadcast_to(amp, lead)))


def is_design(t) -> bool:
    """A design term: its coef is a 2-D X [N][K] (see ``Term``)."""
    return t.coef is not None and np.ndim(t.coef) == 2


def is_latent(p) -> bool:
    """A Normal / StudentT prior with a Linear location or one scale per element: ``lower`` makes it a latent factor."""
    if p.dist not in LINEAR_PRIORS or len(p.params) != PRIOR_DISTS[p.dist][1]:
        return False
    loc, scale = LINEAR_PRIORS[p.dist]
    return isinstance(p.params[loc], Linear) or (not isinstance(p.params[scale], Ref) and np.ndim(p.params[scale]) == 1)


@dataclass(frozen=True)
class Ref:
    """A parameter that is another (scalar) value variable, seen through its transform (e.g. sigma_a)."""

    var: str


@dataclass
class Var:
    name: str          # value-variable name as PyMC names it: "{rv}_{transform}__" (model/core.py:2141-2153)
    rv_name: str
    size: int
    transform: str | None = None
    bounds: tuple[float, float] | None = None
    initial: np.ndarray | float | None = None  # unconstrained support point (pymc/initial_point.py); default 0


@dataclass
class Prior:
    dist: str
    var: str
    params: tuple = ()


@dataclass
class Spectral:
    """The spectral description of an HSGP term: s_k = amplitude * sqrt(S(omega_k; ls)) with S the power spectral density
    of ``cov`` ("expquad", "matern52" or "matern32") at the frequencies omega [M][D] (``hsgp_basis``).  ``ls`` is a constant
    > 0, D constants or a Ref to a variable of size 1 (isotropic) or D (ARD) with positive support; ``amplitude`` (PyMC's
    eta of ``eta**2 * cov``) is a constant > 0 or a Ref to a scalar with positive support."""

    cov: str
    omega: np.ndarray
    ls: float | np.ndarray | Ref = 1.0
    amplitude: float | Ref = 1.0


@dataclass
class Term:
    """coef[i] * prod_f x_f[idx_f[i]].  A factor's idx is None for a scalar variable (broadcast) or for a vector variable of
    the likelihood's own length (elementwise).

    A design term has a 2-D coef X of shape [N][K] and exactly one factor, a variable of size K with no index:
    it adds sum_k X[i, k] * x[k], i.e. ``pm.math.dot(X, beta)``, evaluated on the device as one team-parallel term.

    A spectral term is a design term with a ``spectral`` description: coef is the HSGP basis Phi [N][M], its factor the
    coefficients z (size M, no transform), and it adds sum_k Phi[i, k] s_k(theta) z_k, ``phi @ (beta * sqrt_psd)``."""

    factors: list  # [(var_name, idx or None), ...]
    coef: np.ndarray | float | None = None
    spectral: Spectral | None = None


@dataclass
class Linear:
    """The location of a Normal / StudentT prior as a linear predictor of the CONSTRAINED variables, in the closed form of a
    likelihood's location: mu_j = sum_t coef_t[j] * prod_f x_f[idx_f[j]] with j over the elements of the prior's variable
    (``Term``s, design terms included).  ``a ~ Normal(g0 + g1 * u + r[region], sigma_a)`` is
    ``Prior("normal", "a", (Linear([Term([("g0", None)]), Term([("g1", None)], coef=u), Term([("r", region)])]), Ref(...)))``."""

    terms: list


@dataclass
class Likelihood:
    dist: str
    y: np.ndarray
    terms: list
    sigma: float | Ref | np.ndarray | None = None
    nu: float = 0.0
    name: str = "y"
    alpha: float | Ref | None = None           # negative_binomial_log / gamma_log: dispersion (shape); Weibull: shape
    trials: float | np.ndarray | None = None   # binomial_logit: number of trials, one for all or one per observation
    lower: float | np.ndarray | None = None    # censored / truncated: None (open), a constant or one per observation,
    upper: float | np.ndarray | None = None    # -inf / +inf where that observation's side is open (survival: lower 0 too)
    cutpoints: Ref | np.ndarray | None = None  # ordered_logistic / ordered_probit: K - 1 cutpoints (see ORDINAL_LIKS)
    psi: float | Ref | Linear | None = None    # the zero-inflated / hurdle likelihoods (ZI_LIKS): a Linear is logit(psi)
    weights: Ref | np.ndarray | None = None     # mixtures (MIXTURE_LIKS): a simplex variable or K constants
    components: Ref | np.ndarray | None = None  # mixtures: mu_k (normal_mixture) or lam_k (poisson_mixture)
    phi: float | Ref | None = None              # BETA_LIKS: the precision, PyMC's nu of Beta(mu, nu)

    def n_components(self, model: "ModelIR") -> int:
        """K of a mixture: the size of its components."""
        if isinstance(self.components, Ref):
            return model.var(self.components.var).size
        return int(np.size(self.components))

    def n_categories(self, model: "ModelIR") -> int:
        """K of an ordinal likelihood: one more than its number of cutpoints."""
        if isinstance(self.cutpoints, Ref):
            return model.var(self.cutpoints.var).size + 1
        return int(np.size(self.cutpoints)) + 1

    def bounds(self) -> tuple[np.ndarray, np.ndarray]:
        """(lower, upper) of every observation as float arrays, -inf / +inf where open."""
        N = len(self.y)
        lo = np.full(N, -np.inf) if self.lower is None else np.broadcast_to(np.asarray(self.lower, dtype=np.float64), (N,))
        hi = np.full(N, np.inf) if self.upper is None else np.broadcast_to(np.asarray(self.upper, dtype=np.float64), (N,))
        return np.array(lo), np.array(hi)


@dataclass
class Deterministic:
    """``pm.Deterministic(name, expr)`` whose expression is a linear predictor of the CONSTRAINED variables (the same closed form as
    a likelihood's location): recorded in the posterior group like the reference's trace does (model/core.py:1956-2040,
    backends/base.py:184-191), evaluated on the host from the draws -- it never enters logp."""

    name: str
    size: int
    terms: list
    probs_of: str | None = None  # the {name}_probs of ordinal likelihood `probs_of`: [N, K] category probabilities, from
                                 # that likelihood's eta, cutpoints and sigma (terms unused)


def ordinal_log_probs(dist: str, eta, cutpoints, sigma=1.0) -> np.ndarray:
    """log P(y = k | eta) for k = 0..K-1 along a new last axis: OrderedLogistic / OrderedProbit.compute_p
    (discrete.py:1312-1326, :1416-1432) in log space, as the difference of upper tails above the mode and of lower ones below."""
    from scipy.special import log_ndtr

    c = np.asarray(cutpoints, dtype=np.float64)
    eta, s = np.asarray(eta, dtype=np.float64)[..., None], np.asarray(sigma, dtype=np.float64)[..., None]
    inf = np.full(c.shape[:-1] + (1,), np.inf)
    a = (np.concatenate([-inf, c], axis=-1) - eta) / s  # [..., N, K]
    b = (np.concatenate([c, inf], axis=-1) - eta) / s
    log_cdf = (lambda t: -np.logaddexp(0.0, -t)) if dist == "ordered_logistic" else log_ndtr
    with np.errstate(divide="ignore", invalid="ignore"):
        upper = log_cdf(-a) + np.log1p(-np.exp(log_cdf(-b) - log_cdf(-a)))
        lower = log_cdf(b) + np.log1p(-np.exp(log_cdf(a) - log_cdf(b)))
    return np.where(a > 0, upper, lower)


@dataclass
class AR1:
    var: str
    phi: float | Ref = 1.0
    sigma: float | Ref = 1.0
    init_sigma: float = 1.0


@dataclass
class ModelIR:
    vars: list
    priors: list = field(default_factory=list)
    likelihoods: list = field(default_factory=list)
    ar1: list = field(default_factory=list)
    name: str = "model"
    deterministics: list = field(default_factory=list)

    # ---- layout -----------------------------------------------------------------------------------------------------
    @property
    def n(self) -> int:
        return sum(v.size for v in self.vars)

    def offsets(self) -> dict:
        out, off = {}, 0
        for v in self.vars:
            out[v.name] = off
            off += v.size
        return out

    def var(self, name: str) -> Var:
        for v in self.vars:
            if v.name == name or v.rv_name == name:
                return v
        raise KeyError(name)

    def initial_point(self) -> np.ndarray:
        q = np.zeros(self.n)
        off = self.offsets()
        for v in self.vars:
            if v.initial is not None:
                q[off[v.name] : off[v.name] + v.size] = v.initial
        return q

    def validate(self) -> None:
        names = [v.name for v in self.vars]
        if len(set(names)) != len(names):
            raise ValueError("duplicate value-variable names")
        for v in self.vars:
            if v.transform not in TRANSFORMS:
                raise ValueError(f"{v.name}: transform {v.transform!r} is not in the closed set {list(TRANSFORMS)}")
            if v.transform == "interval" and not (v.bounds and v.bounds[0] < v.bounds[1]):
                raise ValueError(f"{v.name}: interval transform needs bounds lo < hi")
            if v.size < 1:
                raise ValueError(f"{v.name}: size must be positive")
        self._validate_simplex_use()
        n_simplex_priors = {}
        for p in self.priors:
            if p.dist not in PRIOR_DISTS:
                raise ValueError(f"prior {p.dist!r} is not in the closed set {sorted(PRIOR_DISTS)}")
            if len(p.params) != PRIOR_DISTS[p.dist][1]:
                raise ValueError(f"prior {p.dist} on {p.var}: expected {PRIOR_DISTS[p.dist][1]} parameters")
            v = self.var(p.var)
            if v.transform == "simplex" or p.dist == "dirichlet":
                self._check_dirichlet(p, v, n_simplex_priors)
                continue
            loc, scale = LINEAR_PRIORS.get(p.dist, (None, None))
            for k, a in enumerate(p.params):
                what = f"prior {p.dist} on {v.name}"
                if isinstance(a, Linear):
                    if k != loc:
                        raise ValueError(f"{what}: parameter {k} cannot be a Linear predictor (only the location of a "
                                         f"normal or studentt prior can)")
                    self._check_terms(a.terms, v.size, f"{what}: location", "its variable's size")
                    continue
                if isinstance(a, Ref):
                    if self.var(a.var).size != 1:
                        raise ValueError(f"prior on {p.var}: parameter {a.var} must be a scalar variable")
                    if p.dist in ("uniform", "gamma", "beta", "inversegamma") or (p.dist == "studentt" and k == 0):
                        raise ValueError(f"prior {p.dist} on {p.var}: parameter {k} must be a constant")
                if k == scale and not isinstance(a, Ref) and np.ndim(a) == 1:  # one scale per element
                    s = np.asarray(a, dtype=np.float64)
                    if len(s) != v.size or not (np.all(np.isfinite(s)) and np.all(s > 0)):
                        raise ValueError(f"{what}: sigma per element must be a finite constant > 0 for each of the "
                                         f"{v.size} elements")
                    continue
                if k in SCALE_PARAMS.get(p.dist, {}):
                    self._check_scale(a, f"{what}: {SCALE_PARAMS[p.dist][k]}")
            self._check_prior_support(p, v)
        for v in self.vars:
            if v.transform == "simplex" and n_simplex_priors.get(v.name, 0) != 1:
                raise ValueError(f"{v.name}: {SIMPLEX_PRIOR}")
        for L in self.likelihoods:
            if L.dist not in LIK_DISTS:
                raise ValueError(f"likelihood {L.dist!r} is not in the closed set {sorted(LIK_DISTS)}")
            N = len(L.y)
            self._check_terms(L.terms, N, f"likelihood {L.name}", "the number of observations")
            if L.dist in MIXTURE_LIKS:
                self._validate_mixture(L)
                continue
            if L.dist in BETA_LIKS:
                self._validate_beta(L)
                continue
            if L.phi is not None:
                raise ValueError(f"{L.dist} likelihood {L.name}: phi belongs to the beta_logit / beta_binomial_logit "
                                 "likelihoods")
            if L.weights is not None or L.components is not None:
                raise ValueError(f"{L.dist} likelihood {L.name}: weights and components belong to the mixture likelihoods")
            if L.dist in SIGMA_LIKS and L.sigma is None:
                raise ValueError(f"{L.dist} likelihood needs sigma")
            if isinstance(L.sigma, Ref) and self.var(L.sigma.var).size != 1:
                raise ValueError("likelihood sigma must be a scalar variable")
            if L.dist in SIGMA_LIKS:
                if not isinstance(L.sigma, Ref) and np.ndim(L.sigma) == 1:
                    s = np.asarray(L.sigma, dtype=np.float64)
                    if len(s) != N:
                        raise ValueError(f"{L.dist} likelihood {L.name}: sigma must be a scalar or one per observation")
                    if not (np.all(np.isfinite(s)) and np.all(s > 0)):
                        raise ValueError(f"{L.dist} likelihood {L.name}: sigma must be a finite constant > 0 for every observation")
                else:
                    self._check_scale(L.sigma, f"{L.dist} likelihood {L.name}: sigma")
            if L.dist == "studentt" and not (np.isfinite(L.nu) and L.nu > 0):
                raise ValueError(f"studentt likelihood {L.name}: StudentT nu must be > 0")
            y = np.asarray(L.y, dtype=np.float64)
            if L.dist == "poisson_log" and not (np.all(np.isfinite(y)) and np.all(y == np.floor(y)) and np.all(y >= 0)):
                raise ValueError("poisson_log: y must be integers >= 0")
            if L.dist == "bernoulli_logit" and not np.all((y == 0.0) | (y == 1.0)):
                raise ValueError("bernoulli_logit: y must be 0 or 1")
            self._validate_family(L)
            self._validate_bounds(L)
            self._validate_ordinal(L)
            self._validate_psi(L)
            self._validate_survival(L)
        for a in self.ar1:
            if self.var(a.var).size < 2:
                raise ValueError("AR1 needs at least two steps")
            for r in (a.phi, a.sigma):
                if isinstance(r, Ref) and self.var(r.var).size != 1:
                    raise ValueError("AR1 parameters must be scalar variables or constants")
            self._check_scale(a.sigma, f"AR1 on {a.var}: sigma")
            if not (np.isfinite(a.init_sigma) and a.init_sigma > 0):
                raise ValueError(f"AR1 on {a.var}: init_sigma must be > 0")

    def _validate_simplex_use(self) -> None:
        """A simplex variable is used only as a mixture's weights: never as a parameter, a term factor (of a likelihood, a
        Linear location, logit(psi) or a Deterministic), cutpoints, psi, a mixture's components or sigma, or in an AR(1)."""
        simplex = {v.name for v in self.vars if v.transform == "simplex"}
        if not simplex:
            return
        used = []

        def terms(ts):
            used.extend(vn for t in ts for vn, _ in t.factors)

        def par(a):
            if isinstance(a, Ref):
                used.append(a.var)
            elif isinstance(a, Linear):
                terms(a.terms)

        for p in self.priors:
            for a in p.params:
                par(a)
        for L in self.likelihoods:
            terms(L.terms)
            for a in (L.sigma, L.alpha, L.psi, L.cutpoints, L.components, L.phi):
                par(a)
        for a in self.ar1:
            used.append(a.var)
            par(a.phi)
            par(a.sigma)
        for d in self.deterministics:
            terms(d.terms)
        if any(self.var(vn).name in simplex for vn in used):
            raise ValueError(SIMPLEX_USE)

    def _check_dirichlet(self, p, v, count: dict) -> None:
        """A prior on a simplex variable is its one Dirichlet; a Dirichlet sits on a simplex variable and its a is one
        constant > 0, or K equal ones (the checks prepare_ir makes, in the same words)."""
        what = f"prior {p.dist} on {v.name}"
        if v.transform == "simplex":
            if p.dist != "dirichlet" or count.get(v.name, 0) > 0:
                raise ValueError(f"{what}: {SIMPLEX_PRIOR}")
            count[v.name] = 1
        if v.transform != "simplex":
            raise ValueError(f"{what}: {DIRICHLET_VAR}")
        a = p.params[0]
        if isinstance(a, (Ref, Linear)):
            raise ValueError(f"{what}: {DIRICHLET_A}")
        a = np.asarray(a, dtype=np.float64)
        if not (a.ndim == 0 or (a.ndim == 1 and len(a) == v.size + 1)) or not (np.all(np.isfinite(a)) and np.all(a > 0)) \
                or np.any(a != a.ravel()[0]):
            raise ValueError(f"{what}: {DIRICHLET_A}")

    def _validate_mixture(self, L) -> None:
        """K, y, weights, components and sigma of a mixture (the checks prepare_ir makes, in the same words)."""
        what = f"{L.dist} likelihood {L.name}"
        normal = L.dist == "normal_mixture"
        if any(a is not None for a in (L.alpha, L.trials, L.lower, L.upper, L.cutpoints, L.psi)) or \
                (not normal and L.sigma is not None):
            raise ValueError(f"{what}: {MIX_SLOTS}")
        comp_words = MIX_MU if normal else MIX_LAM
        if L.components is None or not (isinstance(L.components, Ref) or np.ndim(L.components) == 1):
            raise ValueError(f"{what}: {comp_words}")
        K = L.n_components(self)
        if K < 2:
            raise ValueError(f"{what}: {MIX_K}")
        y = np.asarray(L.y, dtype=np.float64)
        if normal and not np.all(np.isfinite(y)):
            raise ValueError(f"{what}: {MIX_Y_NORMAL}")
        if not normal and not (np.all(np.isfinite(y)) and np.all(y == np.floor(y)) and np.all(y >= 0)):
            raise ValueError(f"{what}: {ZI_Y}")
        w = L.weights
        if isinstance(w, Ref):
            v = self.var(w.var)
            if not (v.transform == "simplex" and v.size == K - 1):
                raise ValueError(f"{what}: {MIX_WEIGHTS}")
        else:
            wa = None if w is None else np.asarray(w, dtype=np.float64)
            if wa is None or wa.shape != (K,) or not (np.all(np.isfinite(wa)) and np.all(wa >= 0)) or not np.isclose(wa.sum(), 1.0):
                raise ValueError(f"{what}: {MIX_WEIGHTS}")
        c = L.components
        if isinstance(c, Ref):
            v = self.var(c.var)
            ok = v.size == K and (v.transform in (None, "ordered") if normal else _positive_support(v))
        else:
            ca = np.asarray(c, dtype=np.float64)
            ok = bool(np.all(np.isfinite(ca)) and (normal or np.all(ca > 0)))
        if not ok:
            raise ValueError(f"{what}: {comp_words}")
        if normal:
            s = L.sigma
            if isinstance(s, Ref):
                v = self.var(s.var)
                ok = v.size in (1, K) and _positive_support(v)
            else:
                sa = None if s is None else np.asarray(s, dtype=np.float64)
                ok = sa is not None and sa.shape in ((), (K,)) and bool(np.all(np.isfinite(sa)) and np.all(sa > 0))
            if not ok:
                raise ValueError(f"{what}: {MIX_SIGMA}")

    def _validate_beta(self, L) -> None:
        """phi, y and trials of Beta / BetaBinomial observations (the checks prepare_ir makes, in the same words)."""
        what = f"{L.dist} likelihood {L.name}"
        if any(a is not None for a in (L.sigma, L.alpha, L.cutpoints, L.psi, L.weights, L.components, L.lower, L.upper)):
            raise ValueError(f"{what}: {BETA_SLOTS}")
        if L.dist == "beta_logit" and L.trials is not None:
            raise ValueError(f"{what}: {BETA_TRIALS}")
        if L.phi is None:
            raise ValueError(f"{L.dist} needs phi")
        if isinstance(L.phi, Ref) and self.var(L.phi.var).size != 1:
            raise ValueError(f"{L.dist}: phi must be a scalar variable")
        if isinstance(L.phi, Linear) or (not isinstance(L.phi, Ref) and np.ndim(L.phi) != 0):
            raise ValueError(f"{what}: phi must be one constant or a scalar variable")
        self._check_scale(L.phi, f"{what}: phi")
        y = np.asarray(L.y, dtype=np.float64)
        if L.dist == "beta_logit":
            if not (np.all(np.isfinite(y)) and np.all((y > 0.0) & (y < 1.0))):
                raise ValueError(f"{what}: {BETA_Y}")
            return
        if L.trials is None or isinstance(L.trials, (Ref, Linear)):
            raise ValueError(f"{what}: trials must be a constant scalar or a constant array")
        n = np.asarray(L.trials, dtype=np.float64)
        if n.ndim > 1 or (n.ndim == 1 and len(n) != len(y)):
            raise ValueError(f"{what}: trials must be a scalar or one per observation")
        n = np.broadcast_to(n, y.shape)
        if not (np.all(np.isfinite(n)) and np.all(n == np.floor(n)) and np.all(n >= 0)):
            raise ValueError(f"{what}: {BB_TRIALS}")
        if not (np.all(np.isfinite(y)) and np.all(y == np.floor(y)) and np.all((y >= 0) & (y <= n))):
            raise ValueError(f"{what}: {ZIB_Y}")

    def _check_terms(self, terms, N: int, where: str, length: str) -> None:
        """Terms of a predictor of length N (a likelihood's observations, or the elements of a prior's variable)."""
        for t in terms:
            if t.spectral is not None:
                self._check_spectral(t, N, where)
                continue
            if is_design(t):
                self._check_design(t, N, where)
                continue
            if len(t.factors) > MAX_TERM_FACTORS:  # no factor: a constant offset coef[i]
                raise ValueError(f"{where}: a term has at most {MAX_TERM_FACTORS} variable factors")
            for vn, idx in t.factors:
                v = self.var(vn)
                if idx is None and v.size not in (1, N):
                    raise ValueError(f"{where}: {vn} (size {v.size}) needs an index array to enter a predictor of length {N}")
                if idx is not None and len(idx) != N:
                    raise ValueError(f"{where}: the index of {vn} has length {len(idx)}, not {length} {N}")
                if idx is not None and (np.min(idx) < 0 or np.max(idx) >= v.size):
                    raise ValueError(f"{where}: index of {vn} out of range")
            if t.coef is not None and np.ndim(t.coef) == 1 and len(t.coef) != N:
                raise ValueError(f"{where}: coef length {len(t.coef)} differs from {length} {N}")

    def _check_design(self, t, N: int, where: str) -> None:
        """A design term: X [N][K] of finite values, one factor on a variable of size K, no index (the checks prepare_ir
        makes, in the same words)."""
        if len(t.factors) != 1:
            raise ValueError(f"{where}: a design term has exactly one factor (got {len(t.factors)})")
        vn, idx = t.factors[0]
        if idx is not None:
            raise ValueError(f"{where}: a design term's factor takes no index ({vn})")
        X = np.asarray(t.coef)
        K = self.var(vn).size
        if X.shape != (N, K):
            raise ValueError(f"{where}: X must have shape (N, size of the variable): X is {X.shape}, N = {N}, {vn} has size {K}")
        if not np.all(np.isfinite(X)):
            raise ValueError(f"{where}: X must be finite")

    def _check_spectral(self, t, N: int, where: str) -> None:
        """A spectral term: Phi [N][M] finite on one whole variable z of size M with no index and no transform, a known cov,
        omega [M][D], ls and amplitude (the checks prepare_ir makes, in the same words)."""
        sp = t.spectral
        if len(t.factors) != 1:
            raise ValueError(f"{where}: {SPEC_Z}")
        vn, idx = t.factors[0]
        v = self.var(vn)
        if idx is not None or v.transform is not None:
            raise ValueError(f"{where}: {SPEC_Z}")
        Phi = np.asarray(t.coef, dtype=np.float64)
        if Phi.shape != (N, v.size) or not np.all(np.isfinite(Phi)):
            raise ValueError(f"{where}: {SPEC_PHI}")
        if sp.cov not in COV_FUNCS:
            raise ValueError(f"{where}: {SPEC_COV}")
        om = np.asarray(sp.omega, dtype=np.float64)
        if om.ndim != 2 or om.shape[0] != v.size or not 1 <= om.shape[1] <= 4096 or not (
                np.all(np.isfinite(om)) and np.all(om >= 0)):
            raise ValueError(f"{where}: {SPEC_OMEGA}")
        D = om.shape[1]

        def ok(a, sizes, shapes):  # a Ref to a variable of one of the sizes with positive support, or constants > 0
            if isinstance(a, Ref):
                w = self.var(a.var)
                return w.size in sizes and _positive_support(w)
            if isinstance(a, Linear):
                return False
            c = np.asarray(a, dtype=np.float64)
            return c.shape in shapes and bool(np.all(np.isfinite(c)) and np.all(c > 0))

        if not ok(sp.amplitude, (1,), ((),)):
            raise ValueError(f"{where}: {SPEC_AMP}")
        if not ok(sp.ls, (1, D), ((), (D,))):
            raise ValueError(f"{where}: {SPEC_LS}")

    def _check_scale(self, a, what: str) -> None:
        """A scale slot (a prior's sigma / beta / lam, a likelihood's sigma, an AR(1) sigma, a dispersion alpha): a finite
        constant > 0, or a Ref to a scalar variable whose transform keeps it positive."""
        if isinstance(a, Ref):
            v = self.var(a.var)
            if v.size == 1 and _positive_support(v):
                return
        elif np.ndim(a) == 0 and np.isfinite(float(a)) and float(a) > 0:
            return
        raise ValueError(f"{what} must be a finite constant > 0 or {POSITIVE_SUPPORT}")

    def _check_prior_support(self, p, v) -> None:
        """The variable's transform keeps it inside the prior's support; the constant parameters are in their domain."""
        lo, hi = v.bounds if v.transform == "interval" else (None, None)
        if v.transform in ORDERED_TRANSFORMS and not (
                p.dist in REAL_LINE_PRIORS or (p.dist in POSITIVE_PRIORS and v.transform == "ordered_positive")):
            raise ValueError(f"prior {p.dist} on {v.name}: {ORDERED_PRIOR}")
        if p.dist in POSITIVE_PRIORS and not _positive_support(v):
            raise ValueError(f"prior {p.dist} on {v.name}: the variable needs a log transform or an interval with lo >= 0 "
                             "(positive support)")
        if p.dist == "studentt" and not (np.isfinite(float(p.params[0])) and float(p.params[0]) > 0):
            raise ValueError(f"prior studentt on {v.name}: StudentT nu must be a positive constant")
        if p.dist in ("gamma", "beta") and not all(np.isfinite(float(a)) and float(a) > 0 for a in p.params):
            raise ValueError(f"prior {p.dist} on {v.name}: {p.dist.capitalize()} needs constant alpha, beta > 0")
        if p.dist == "inversegamma" and not all(np.isfinite(float(a)) and float(a) > 0 for a in p.params):
            raise ValueError(f"prior inversegamma on {v.name}: InverseGamma needs constant alpha, beta > 0")
        if p.dist == "beta" and not (lo is not None and lo >= 0.0 and hi <= 1.0):
            raise ValueError(f"prior beta on {v.name}: the variable needs an interval inside [0, 1]")
        if p.dist == "uniform":
            a, b = float(p.params[0]), float(p.params[1])
            if not a < b:
                raise ValueError(f"prior uniform on {v.name}: Uniform bounds must be constants lo < hi")
            if not (lo is not None and lo >= a and hi <= b):
                raise ValueError(f"prior uniform on {v.name}: the variable needs an interval inside the Uniform bounds")

    def _validate_family(self, L) -> None:
        """Support and parameter rules of the count / positive families (the same checks prepare_ir makes)."""
        y = np.asarray(L.y, dtype=np.float64)
        integer = lambda a: bool(np.all(np.isfinite(a)) and np.all(a == np.floor(a)))  # noqa: E731
        fam = ZI_FAMILY.get(L.dist, L.dist)  # a zero-inflated / hurdle likelihood follows its family's rules
        if L.dist in ("zero_inflated_poisson", "hurdle_poisson"):
            if not integer(y) or np.any(y < 0):
                raise ValueError(f"{L.dist}: {ZI_Y}")
            if L.sigma is not None:
                raise ValueError(f"{L.dist}: {ZIP_SLOT}")
        if fam == "binomial_logit":
            if L.trials is None or isinstance(L.trials, Ref):
                raise ValueError("binomial_logit: trials must be a constant scalar or a constant array")
            n = np.asarray(L.trials, dtype=np.float64)
            if n.ndim > 1 or (n.ndim == 1 and len(n) != len(y)):
                raise ValueError("binomial_logit: trials must be a scalar or one per observation")
            if not integer(n) or np.any(n < 0):
                raise ValueError("binomial_logit: trials must be integers >= 0")
            if not integer(y) or np.any(y < 0) or np.any(y > n):
                raise ValueError(f"{L.dist}: {ZIB_Y}")
        elif L.trials is not None:
            raise ValueError(f"{L.dist}: trials belong to binomial_logit")
        if fam in DISPERSION_LIKS:
            if L.alpha is None:
                raise ValueError(f"{L.dist} needs alpha")
            if isinstance(L.alpha, Ref) and self.var(L.alpha.var).size != 1:
                raise ValueError(f"{L.dist}: alpha must be a scalar variable")
            self._check_scale(L.alpha, f"{L.dist}: alpha")
            if fam == "negative_binomial_log" and (not integer(y) or np.any(y < 0)):
                raise ValueError(f"{L.dist}: {ZI_Y}")
            if L.dist == "gamma_log" and not (np.all(np.isfinite(y)) and np.all(y > 0)):
                raise ValueError("gamma_log: y must be > 0")
            if L.dist == "hurdle_gamma" and not (np.all(np.isfinite(y)) and np.all(y >= 0)):
                raise ValueError(f"hurdle_gamma: {HG_Y}")
        elif L.alpha is not None and L.dist not in WEIBULL_LIKS:
            raise ValueError(f"{L.dist}: alpha belongs to the negative_binomial_log / gamma_log likelihoods")
        if fam in ("binomial_logit",) + DISPERSION_LIKS and L.sigma is not None:
            raise ValueError(f"{L.dist} has no sigma (its parameter is {'trials' if L.dist == 'binomial_logit' else 'alpha'})")

    def _validate_bounds(self, L) -> None:
        """Bounds of censored / truncated Normal observations (the checks prepare_ir makes, in the same words)."""
        what = f"{L.dist} likelihood {L.name}"
        if L.dist in SURVIVAL_LIKS:  # _validate_survival
            return
        if L.dist not in BOUNDED_LIKS:
            if L.lower is not None or L.upper is not None:
                raise ValueError(f"{what}: lower / upper belong to the censored_normal / truncated_normal likelihoods")
            return
        N = len(L.y)
        for side in (L.lower, L.upper):
            if isinstance(side, Ref):
                raise ValueError(f"{what}: lower and upper are data (None, a constant or one per observation), not variables")
            if side is not None and not (np.ndim(side) == 0 or (np.ndim(side) == 1 and len(side) == N)):
                raise ValueError(f"{what}: lower and upper must be None, a constant or one value per observation (N = {N})")
        lo, hi = L.bounds()
        y = np.asarray(L.y, dtype=np.float64)
        if np.any(np.isnan(lo) | np.isnan(hi) | (lo == np.inf) | (hi == -np.inf)):
            raise ValueError(f"{what}: {BOUND_SIDES}")
        if not np.all(lo < hi):
            raise ValueError(f"{what}: {BOUND_ORDER}")
        if not (np.all(np.isfinite(y)) and np.all((lo <= y) & (y <= hi))):
            raise ValueError(f"{what}: {BOUND_Y}")
        if L.dist == "truncated_normal" and not np.any(np.isfinite(lo) | np.isfinite(hi)):
            raise ValueError(f"{what}: {TRUNC_OPEN}")

    def _validate_survival(self, L) -> None:
        """y, bounds and the shape alpha of Weibull / LogNormal observations (the checks prepare_ir makes, in the same
        words).  A lower bound of 0 is an open side, as -inf is: every y is > 0."""
        if L.dist not in SURVIVAL_LIKS:
            return
        what = f"{L.dist} likelihood {L.name}"
        if L.dist in WEIBULL_LIKS:
            if L.alpha is None:
                raise ValueError(f"{L.dist} needs alpha")
            if isinstance(L.alpha, Ref) and self.var(L.alpha.var).size != 1:
                raise ValueError(f"{L.dist}: alpha must be a scalar variable")
            if not isinstance(L.alpha, Ref) and np.ndim(L.alpha) != 0:
                raise ValueError(f"{what}: alpha must be one constant or a scalar variable")
            self._check_scale(L.alpha, f"{L.dist}: alpha")
            if L.sigma is not None:
                raise ValueError(f"{what}: {WEIBULL_SIGMA}")
        y = np.asarray(L.y, dtype=np.float64)
        if not (np.all(np.isfinite(y)) and np.all(y > 0)):
            raise ValueError(f"{what}: {SURV_Y}")
        if L.dist not in SURVIVAL_BOUNDED:
            if L.lower is not None or L.upper is not None:
                raise ValueError(f"{what}: {SURV_PLAIN}")
            return
        N = len(y)
        for side in (L.lower, L.upper):
            if isinstance(side, Ref):
                raise ValueError(f"{what}: lower and upper are data (None, a constant or one per observation), not variables")
            if side is not None and not (np.ndim(side) == 0 or (np.ndim(side) == 1 and len(side) == N)):
                raise ValueError(f"{what}: lower and upper must be None, a constant or one value per observation (N = {N})")
        lo, hi = L.bounds()
        if np.any(np.isnan(lo) | np.isnan(hi) | ~((lo >= 0) | (lo == -np.inf)) | (lo == np.inf) | ~(hi > 0)):
            raise ValueError(f"{what}: {SURV_SIDES}")
        if not np.all(lo < hi):
            raise ValueError(f"{what}: {BOUND_ORDER}")
        if not np.all((lo <= y) & (y <= hi)):
            raise ValueError(f"{what}: {BOUND_Y}")
        if L.dist.startswith("truncated") and not np.any((np.isfinite(lo) & (lo > 0)) | np.isfinite(hi)):
            raise ValueError(f"{what}: {SURV_TRUNC_OPEN}")

    def _validate_ordinal(self, L) -> None:
        """Cutpoints and categories of ordinal observations (the checks prepare_ir makes, in the same words)."""
        what = f"{L.dist} likelihood {L.name}"
        if L.dist not in ORDINAL_LIKS:
            if L.cutpoints is not None:
                raise ValueError(f"{what}: cutpoints belong to the ordered_logistic / ordered_probit likelihoods")
            return
        if L.dist == "ordered_logistic" and L.sigma is not None:
            raise ValueError(f"{what}: {LOGISTIC_SIGMA}")
        if L.cutpoints is None:
            raise ValueError(f"{what}: needs cutpoints")
        if isinstance(L.cutpoints, Ref):
            v = self.var(L.cutpoints.var)
            if v.size > 1 and v.transform not in ORDERED_TRANSFORMS:
                raise ValueError(f"{what}: {CUT_ORDERED}")
        else:
            c = np.asarray(L.cutpoints, dtype=np.float64)
            if c.ndim != 1 or not (np.all(np.isfinite(c)) and np.all(np.diff(c) > 0)):
                raise ValueError(f"{what}: {CUT_CONST}")
        K = L.n_categories(self)
        if K < 2:
            raise ValueError(f"{what}: {ORD_K}")
        y = np.asarray(L.y, dtype=np.float64)
        if not (np.all(np.isfinite(y)) and np.all(y == np.floor(y)) and np.all((y >= 0) & (y <= K - 1))):
            raise ValueError(f"{what}: {ORD_Y}")

    def _validate_psi(self, L) -> None:
        """psi of zero-inflated / hurdle observations (the checks prepare_ir makes, in the same words)."""
        what = f"{L.dist} likelihood {L.name}"
        if L.dist not in ZI_LIKS:
            if L.psi is not None:
                raise ValueError(f"{what}: psi belongs to the zero-inflated and hurdle likelihoods")
            return
        psi = L.psi
        if psi is None:
            raise ValueError(f"{what}: needs psi")
        if isinstance(psi, Linear):
            if not psi.terms:
                raise ValueError(f"{what}: {PSI_BLOCK}")
            self._check_terms(psi.terms, len(L.y), f"{what}: logit(psi)", "the number of observations")
        elif isinstance(psi, Ref):
            v = self.var(psi.var)
            if not (v.size == 1 and v.transform == "interval" and v.bounds[0] >= 0.0 and v.bounds[1] <= 1.0):
                raise ValueError(f"{what}: {PSI_VAR}")
        else:
            if np.ndim(psi) != 0:  # one constant per observation is not provided
                raise ValueError(f"{what}: {PSI_BLOCK}")
            if float(psi) == 1.0:
                raise ValueError(f"{what}: {PSI_ONE}")
            if not (np.isfinite(float(psi)) and 0.0 < float(psi) < 1.0):
                raise ValueError(f"{what}: {PSI_CONST}")

    # ---- host-side post-processing (f1): unconstrained draws -> named constrained RVs --------------------------------
    def constrain(self, q: np.ndarray) -> dict:
        out, off = {}, self.offsets()
        for v in self.vars:
            x = q[..., off[v.name] : off[v.name] + v.size]
            if v.transform == "log":
                x = np.exp(x)
            elif v.transform == "interval":
                lo, hi = v.bounds
                s = 1.0 / (1.0 + np.exp(-x))
                x = s * hi + (1.0 - s) * lo
            elif v.transform in ORDERED_TRANSFORMS:
                x = ordered_backward(np.array(x, dtype=np.float64), v.transform == "ordered_positive")
            elif v.transform == "simplex":  # the K weights, as PyMC's posterior holds a Dirichlet
                x = simplex_backward(x)
                out[v.rv_name] = x
                continue
            out[v.rv_name] = x[..., 0] if v.size == 1 else x
        return out

    def eval_deterministics(self, posterior: dict) -> dict:
        """Deterministics from CONSTRAINED draws (``posterior``: rv name -> [..., size] or [...] for scalars, as ``constrain``
        returns them): value_i = sum_t coef_t[i] * prod_f x_f[idx_f[i]]."""
        out = {}
        for d in self.deterministics:
            if d.probs_of is not None:  # an ordinal likelihood's category probabilities, [..., N, K]
                L = next(L for L in self.likelihoods if L.name == d.probs_of)
                eta = np.asarray(dataclasses.replace(self, deterministics=[Deterministic("eta", len(L.y), L.terms)])
                                 .eval_deterministics(posterior)["eta"])
                c = posterior[self.var(L.cutpoints.var).rv_name] if isinstance(L.cutpoints, Ref) else L.cutpoints
                c = np.asarray(c, dtype=np.float64)
                c = c[..., None] if isinstance(L.cutpoints, Ref) and self.var(L.cutpoints.var).size == 1 else c
                s = 1.0 if L.dist == "ordered_logistic" else (
                    np.asarray(posterior[self.var(L.sigma.var).rv_name])[..., None] if isinstance(L.sigma, Ref) else L.sigma)
                lead = eta.shape[:-1]
                out[d.name] = np.exp(ordinal_log_probs(L.dist, eta, np.broadcast_to(c[..., None, :], lead + (1, c.shape[-1])), s))
                continue
            lead = None
            total = 0.0
            for t in d.terms:
                if t.spectral is not None:  # Phi @ (z * s(theta))
                    v = self.var(t.factors[0][0])
                    z = np.asarray(posterior[v.rv_name], dtype=np.float64)
                    z = z[..., None] if v.size == 1 else z
                    b = z * spectral_weights(self, t, posterior)
                    lead = b.shape[:-1]
                    total = total + b @ np.asarray(t.coef, dtype=np.float64).T
                    continue
                if is_design(t):  # X @ x
                    v = self.var(t.factors[0][0])
                    x = np.asarray(posterior[v.rv_name])
                    x = x[..., None] if v.size == 1 else x
                    lead = x.shape[:-1]
                    total = total + x @ np.asarray(t.coef, dtype=np.float64).T
                    continue
                term = 1.0 if t.coef is None else np.asarray(t.coef, dtype=np.float64)
                for vn, idx in t.factors:
                    v = self.var(vn)
                    x = np.asarray(posterior[v.rv_name])
                    if v.size == 1:
                        x = x[..., None]
                    lead = x.shape[:-1]
                    term = term * (x[..., np.asarray(idx)] if idx is not None else x)
                total = total + term
            total = np.asarray(total, dtype=np.float64)
            if lead is not None:
                total = np.broadcast_to(total, lead + (d.size,))
            out[d.name] = total[..., 0] if d.size == 1 else total
        return out

    def observed_data(self) -> dict:
        return {L.name: np.asarray(L.y) for L in self.likelihoods}

    def constant_data(self) -> dict:
        out = {}
        for L in self.likelihoods:
            for k, t in enumerate(L.terms):
                if t.coef is not None and np.ndim(t.coef) in (1, 2):  # 2: a design term's X, a spectral term's Phi
                    out[f"{L.name}_coef{k}"] = np.asarray(t.coef)
                if t.spectral is not None:
                    out[f"{L.name}_omega{k}"] = np.asarray(t.spectral.omega)
                for vn, idx in t.factors:
                    if idx is not None:
                        out[f"{L.name}_{vn}_idx"] = np.asarray(idx)
            if L.trials is not None and np.ndim(L.trials) == 1:
                out[f"{L.name}_trials"] = np.asarray(L.trials)
            for side in ("lower", "upper"):  # per-observation bounds of censored / truncated observations
                if np.ndim(getattr(L, side)) == 1:
                    out[f"{L.name}_{side}"] = np.asarray(getattr(L, side))
            if L.cutpoints is not None and not isinstance(L.cutpoints, Ref):  # constant cutpoints of ordinal observations
                out[f"{L.name}_cutpoints"] = np.asarray(L.cutpoints)
            if isinstance(L.psi, Linear):  # the data of logit(psi) of zero-inflated / hurdle observations
                for k, t in enumerate(L.psi.terms):
                    if t.coef is not None and np.ndim(t.coef) in (1, 2):
                        out[f"{L.name}_psi_coef{k}"] = np.asarray(t.coef)
                    if t.spectral is not None:
                        out[f"{L.name}_psi_omega{k}"] = np.asarray(t.spectral.omega)
                    for vn, idx in t.factors:
                        if idx is not None:
                            out[f"{L.name}_psi_{vn}_idx"] = np.asarray(idx)
            elif L.psi is not None and not isinstance(L.psi, Ref):  # a constant psi
                out[f"{L.name}_psi"] = np.asarray(float(L.psi))
            for part in ("weights", "components"):  # the constant blocks of a mixture
                a = getattr(L, part)
                if a is not None and not isinstance(a, Ref):
                    out[f"{L.name}_{part}"] = np.asarray(a)
        return out


# ------------------------------------------------------------------------------------------------------------------------
# the five BASELINE configs that fit the chain-per-warp / chain-per-CTA engines, written in IR
# ------------------------------------------------------------------------------------------------------------------------
def eight_schools_ir() -> ModelIR:
    from .models import EIGHT_SCHOOLS_SIGMA, EIGHT_SCHOOLS_Y

    J = len(EIGHT_SCHOOLS_Y)
    return ModelIR(
        name="eight_schools",
        vars=[Var("mu", "mu", 1), Var("tau_log__", "tau", 1, "log", initial=np.log(5.0)), Var("theta_t", "theta_t", J)],
        priors=[Prior("normal", "mu", (0.0, 5.0)), Prior("halfcauchy", "tau_log__", (5.0,)),
                Prior("normal", "theta_t", (0.0, 1.0))],
        likelihoods=[Likelihood("normal", EIGHT_SCHOOLS_Y.copy(),
                                [Term([("mu", None)]), Term([("tau_log__", None), ("theta_t", None)])],
                                sigma=EIGHT_SCHOOLS_SIGMA.copy())],
    )


def radon_ir(n_obs: int = 919, n_counties: int = 85, seed: int = 123) -> ModelIR:
    """benchmarks/benchmarks/benchmarks.py:34-45 (non-centred varying intercept and slope; note sigma = 100**2)."""
    from .models import radon_data

    county, floor, y = radon_data(n_obs, n_counties, seed)
    J = n_counties
    l5 = np.log(5.0)
    return ModelIR(
        name="radon",
        vars=[Var("mu_a", "mu_a", 1), Var("sigma_a_log__", "sigma_a", 1, "log", initial=l5), Var("mu_b", "mu_b", 1),
              Var("sigma_b_log__", "sigma_b", 1, "log", initial=l5), Var("a", "a", J), Var("b", "b", J),
              Var("eps_log__", "eps", 1, "log", initial=l5)],
        priors=[Prior("normal", "mu_a", (0.0, 1.0e4)), Prior("halfcauchy", "sigma_a_log__", (5.0,)),
                Prior("normal", "mu_b", (0.0, 1.0e4)), Prior("halfcauchy", "sigma_b_log__", (5.0,)),
                Prior("normal", "a", (0.0, 1.0)), Prior("normal", "b", (0.0, 1.0)), Prior("halfcauchy", "eps_log__", (5.0,))],
        likelihoods=[Likelihood("normal", y, [
            Term([("mu_a", None)]), Term([("sigma_a_log__", None), ("a", county)]),
            Term([("mu_b", None)], coef=floor), Term([("sigma_b_log__", None), ("b", county)], coef=floor)],
            sigma=Ref("eps_log__"))],
    )


def radon_centred_ir(n_obs: int = 800, n_counties: int = 32, n_regions: int = 4, seed: int = 41) -> ModelIR:
    """Centred varying-intercept Radon-shaped model on simulated data, with a group-level predictor and nested groups:
    a_j ~ Normal(g0 + g1 u_j + r[region_j], sigma_a) over counties j, r_k ~ Normal(0, 1) over regions,
    y_i ~ Normal(a[county_i] + b floor_i, sigma_y); g0, g1, b ~ Normal(0, 5), sigma_a, sigma_y ~ HalfNormal(1).
    Every county holds observations (enough of them that the centred form samples without divergences)."""
    rng = np.random.default_rng(seed)
    J = n_counties
    region = (np.arange(J) % n_regions).astype(np.int32)
    u = rng.standard_normal(J)
    county = np.concatenate([np.arange(J), rng.integers(0, J, n_obs - J)]).astype(np.int32)
    floor = (rng.random(n_obs) < 0.3).astype(np.float64)
    r = rng.normal(0.0, 0.5, n_regions)
    a = 1.3 + 0.7 * u + r[region] + 0.3 * rng.standard_normal(J)
    y = a[county] - 0.6 * floor + 0.7 * rng.standard_normal(n_obs)
    return ModelIR(
        name="radon_centred",
        vars=[Var("g0", "g0", 1), Var("g1", "g1", 1), Var("r", "r", n_regions), Var("sigma_a_log__", "sigma_a", 1, "log"),
              Var("a", "a", J), Var("b", "b", 1), Var("sigma_y_log__", "sigma_y", 1, "log")],
        priors=[Prior("normal", "g0", (0.0, 5.0)), Prior("normal", "g1", (0.0, 5.0)), Prior("normal", "r", (0.0, 1.0)),
                Prior("halfnormal", "sigma_a_log__", (1.0,)),
                Prior("normal", "a", (Linear([Term([("g0", None)]), Term([("g1", None)], coef=u), Term([("r", region)])]),
                                      Ref("sigma_a_log__"))),
                Prior("normal", "b", (0.0, 5.0)), Prior("halfnormal", "sigma_y_log__", (1.0,))],
        likelihoods=[Likelihood("normal", y, [Term([("a", county)]), Term([("b", None)], coef=floor)],
                                sigma=Ref("sigma_y_log__"))],
    )


def stochvol_ir(T: int = 3000, seed: int = 4) -> ModelIR:
    from .models import stochvol

    y = stochvol(T, seed).data["y"]
    return ModelIR(
        name="stochvol",
        vars=[Var("mu", "mu", 1), Var("phi_interval__", "phi", 1, "interval", (-1.0, 1.0)),
              Var("sigma_log__", "sigma", 1, "log", initial=np.log(0.1)), Var("h", "h", T)],
        priors=[Prior("normal", "mu", (0.0, 5.0)), Prior("uniform", "phi_interval__", (-1.0, 1.0)),
                Prior("exponential", "sigma_log__", (10.0,))],
        ar1=[AR1("h", Ref("phi_interval__"), Ref("sigma_log__"), 1.0)],
        likelihoods=[Likelihood("normal_logvar", y, [Term([("mu", None)]), Term([("h", None)])])],
    )


def varying_intercept_logistic_ir(n_obs: int = 600, n_groups: int = 12, n_features: int = 3, seed: int = 17) -> ModelIR:
    """A model with NO hand-written kernel (VERDICT r1 next #8):  alpha_g ~ Normal(mu_alpha, sigma_alpha) (centred),
    beta ~ Normal(0, 2.5), y_i ~ Bernoulli(logit_p = alpha[g_i] + x_i . beta)."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, n_groups, n_obs).astype(np.int32)
    X = rng.standard_normal((n_obs, n_features))
    alpha = rng.normal(0.3, 0.8, n_groups)
    beta = rng.normal(0.0, 1.0, n_features)
    eta = alpha[g] + X @ beta
    y = (rng.random(n_obs) < 1.0 / (1.0 + np.exp(-eta))).astype(np.float64)
    terms = [Term([("alpha", g)])] + [Term([("beta", np.full(n_obs, k, dtype=np.int32))], coef=X[:, k].copy())
                                      for k in range(n_features)]
    return ModelIR(
        name="varying_intercept_logistic",
        vars=[Var("mu_alpha", "mu_alpha", 1), Var("sigma_alpha_log__", "sigma_alpha", 1, "log"),
              Var("alpha", "alpha", n_groups), Var("beta", "beta", n_features)],
        priors=[Prior("normal", "mu_alpha", (0.0, 2.0)), Prior("halfnormal", "sigma_alpha_log__", (1.0,)),
                Prior("normal", "alpha", (Ref("mu_alpha"), Ref("sigma_alpha_log__"))), Prior("normal", "beta", (0.0, 2.5))],
        likelihoods=[Likelihood("bernoulli_logit", y, terms)],
    )


def binomial_logit_ir(n_obs: int = 150, n_groups: int = 10, seed: int = 29) -> ModelIR:
    """Varying-intercept binomial regression on simulated data (rat-tumour / seeds shape): a_g ~ Normal(mu, sigma) (centred),
    beta ~ Normal(0, 1), y_i ~ Binomial(trials_i, logit_p = a[g_i] + beta x_i) with 1..40 trials per observation."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, n_groups, n_obs).astype(np.int32)
    x = rng.standard_normal(n_obs)
    trials = rng.integers(1, 41, n_obs).astype(np.float64)
    a = rng.normal(-0.5, 0.7, n_groups)
    eta = a[g] + 0.4 * x
    y = rng.binomial(trials.astype(np.int64), 1.0 / (1.0 + np.exp(-eta))).astype(np.float64)
    return ModelIR(
        name="binomial_logit",
        vars=[Var("mu", "mu", 1), Var("sigma_log__", "sigma", 1, "log"), Var("a", "a", n_groups), Var("beta", "beta", 1)],
        priors=[Prior("normal", "mu", (0.0, 2.0)), Prior("halfnormal", "sigma_log__", (1.0,)),
                Prior("normal", "a", (Ref("mu"), Ref("sigma_log__"))), Prior("normal", "beta", (0.0, 1.0))],
        likelihoods=[Likelihood("binomial_logit", y, [Term([("a", g)]), Term([("beta", None)], coef=x)], trials=trials)],
    )


def negative_binomial_ir(n_obs: int = 300, n_groups: int = 8, seed: int = 31, alpha: float | None = None) -> ModelIR:
    """Hierarchical negative-binomial regression on simulated overdispersed counts: z_g ~ Normal(0, 1) (non-centred),
    beta ~ Normal(0, 1)^2, alpha ~ Exponential(1) (or the constant `alpha`),
    y_i ~ NegativeBinomial(mu = exp(mu_a + sigma_a z[g_i] + x_i . beta), alpha)."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, n_groups, n_obs).astype(np.int32)
    X = rng.standard_normal((n_obs, 2))
    z = rng.standard_normal(n_groups)
    eta = 1.2 + 0.5 * z[g] + X @ np.array([0.3, -0.2])
    a_true = 2.5
    mu = np.exp(eta)
    y = rng.negative_binomial(a_true, a_true / (mu + a_true)).astype(np.float64)
    vars_ = [Var("mu_a", "mu_a", 1), Var("sigma_a_log__", "sigma_a", 1, "log"), Var("z", "z", n_groups), Var("beta", "beta", 2)]
    priors = [Prior("normal", "mu_a", (0.0, 2.0)), Prior("halfnormal", "sigma_a_log__", (1.0,)), Prior("normal", "z", (0.0, 1.0)),
              Prior("normal", "beta", (0.0, 1.0))]
    if alpha is None:
        vars_.append(Var("alpha_log__", "alpha", 1, "log"))
        priors.append(Prior("exponential", "alpha_log__", (1.0,)))
    terms = [Term([("mu_a", None)]), Term([("sigma_a_log__", None), ("z", g)])] + \
        [Term([("beta", np.full(n_obs, k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(2)]
    return ModelIR(name="negative_binomial", vars=vars_, priors=priors,
                   likelihoods=[Likelihood("negative_binomial_log", y, terms,
                                           alpha=Ref("alpha_log__") if alpha is None else float(alpha))])


def gamma_regression_ir(n_obs: int = 200, n_features: int = 3, seed: int = 37, alpha: float | None = None) -> ModelIR:
    """Gamma regression with a log link on simulated positive data: b0 ~ Normal(0, 2), beta ~ Normal(0, 1)^K,
    alpha ~ HalfNormal(2) (or the constant `alpha`), y_i ~ Gamma(alpha, beta = alpha / exp(b0 + x_i . beta))."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n_obs, n_features))
    eta = 0.7 + X @ rng.normal(0.0, 0.4, n_features)
    a_true = 3.0
    y = rng.gamma(a_true, np.exp(eta) / a_true)
    vars_ = [Var("b0", "b0", 1), Var("beta", "beta", n_features)]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "beta", (0.0, 1.0))]
    if alpha is None:
        vars_.append(Var("alpha_log__", "alpha", 1, "log"))
        priors.append(Prior("halfnormal", "alpha_log__", (2.0,)))
    terms = [Term([("b0", None)])] + [Term([("beta", np.full(n_obs, k, dtype=np.int32))], coef=X[:, k].copy())
                                      for k in range(n_features)]
    return ModelIR(name="gamma_regression", vars=vars_, priors=priors,
                   likelihoods=[Likelihood("gamma_log", y, terms, alpha=Ref("alpha_log__") if alpha is None else float(alpha))])


def censored_regression_ir(n_obs: int = 400, n_groups: int = 8, n_features: int = 3, seed: int = 43) -> ModelIR:
    """Tobit-style regression on simulated data: a_g ~ Normal(mu_a, sigma_a) (centred), beta ~ Normal(0, 1)^K as a design
    term, sigma ~ HalfNormal(1), y*_i = a[g_i] + x_i . beta + sigma e_i recorded as y_i = clip(y*_i, lower, upper_i):
    left-censored at one detection limit for all observations and right-censored at each observation's own follow-up limit."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, n_groups, n_obs).astype(np.int32)
    X = rng.standard_normal((n_obs, n_features))
    a = rng.normal(0.5, 0.6, n_groups)
    ystar = a[g] + X @ rng.normal(0.0, 0.7, n_features) + 0.8 * rng.standard_normal(n_obs)
    lower = float(np.quantile(ystar, 0.2))  # the detection limit
    upper = lower + rng.uniform(1.2, 4.0, n_obs)  # follow-up limits
    y = np.clip(ystar, lower, upper)
    return ModelIR(
        name="censored_regression",
        vars=[Var("mu_a", "mu_a", 1), Var("sigma_a_log__", "sigma_a", 1, "log"), Var("a", "a", n_groups),
              Var("beta", "beta", n_features), Var("sigma_log__", "sigma", 1, "log")],
        priors=[Prior("normal", "mu_a", (0.0, 2.0)), Prior("halfnormal", "sigma_a_log__", (1.0,)),
                Prior("normal", "a", (Ref("mu_a"), Ref("sigma_a_log__"))), Prior("normal", "beta", (0.0, 1.0)),
                Prior("halfnormal", "sigma_log__", (1.0,))],
        likelihoods=[Likelihood("censored_normal", y, [Term([("a", g)]), Term([("beta", None)], coef=X)],
                                sigma=Ref("sigma_log__"), lower=lower, upper=upper)],
    )


def truncated_regression_ir(n_obs: int = 300, n_features: int = 2, seed: int = 47) -> ModelIR:
    """Regression on data recorded only above a threshold: b0 ~ Normal(0, 5), beta ~ Normal(0, 1)^K as a design term,
    sigma ~ HalfNormal(1), y_i ~ TruncatedNormal(b0 + x_i . beta, sigma, lower=threshold, upper=upper_i), where a third of the
    observations also carry an upper bound of their own (+inf for the rest)."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n_obs, n_features))
    eta = 0.4 + X @ (rng.normal(0.0, 0.8, n_features) * np.sqrt(2.0 / max(n_features, 2)))  # sd of eta ~ 0.8 for any K
    lower = 0.0
    upper = np.where(rng.random(n_obs) < 1 / 3, rng.uniform(0.5, 2.5, n_obs), np.inf)
    y = np.empty(n_obs)
    for i in range(n_obs):  # rejection sampling from each observation's truncated Normal
        while True:
            v = eta[i] + 1.1 * rng.standard_normal()
            if lower < v < upper[i]:
                y[i] = v
                break
    return ModelIR(
        name="truncated_regression",
        vars=[Var("b0", "b0", 1), Var("beta", "beta", n_features), Var("sigma_log__", "sigma", 1, "log")],
        priors=[Prior("normal", "b0", (0.0, 5.0)), Prior("normal", "beta", (0.0, 1.0)), Prior("halfnormal", "sigma_log__", (1.0,))],
        likelihoods=[Likelihood("truncated_normal", y, [Term([("b0", None)]), Term([("beta", None)], coef=X)],
                                sigma=Ref("sigma_log__"), lower=lower, upper=upper)],
    )


def ordinal_regression_ir(link: str = "logistic", n_obs: int = 300, n_groups: int = 6, n_features: int = 2, K: int = 5,
                          sigma: str | None = None, seed: int = 53) -> ModelIR:
    """Ordinal regression on simulated ratings: z_g ~ Normal(0, 1), sigma_a ~ HalfNormal(1) (non-centred group intercepts
    sigma_a z[g_i]), beta ~ Normal(0, 1)^F as a design term, cutpoints ~ Normal(linspace(-2, 2, K - 1), 5) with the
    ordered transform, y_i ~ OrderedLogistic(eta_i, cutpoints) or OrderedProbit(eta_i, cutpoints, sigma) with sigma the
    constant 1 (``sigma=None`` or "const") or sigma ~ HalfNormal(1) (``sigma="var"``)."""
    if link not in ("logistic", "probit"):
        raise ValueError("link must be 'logistic' or 'probit'")
    rng = np.random.default_rng(seed)
    g = rng.integers(0, n_groups, n_obs).astype(np.int32)
    X = rng.standard_normal((n_obs, n_features))
    eta = rng.normal(0.0, 0.7, n_groups)[g] + X @ rng.normal(0.0, 0.8, n_features)
    mu_c = np.linspace(-2.0, 2.0, K - 1)
    noise = rng.logistic(size=n_obs) if link == "logistic" else rng.standard_normal(n_obs)
    y = np.searchsorted(mu_c + rng.normal(0.0, 0.2, K - 1).cumsum() * 0.3, eta + noise).astype(np.float64)
    z0 = np.concatenate([[mu_c[0]], np.log(np.diff(mu_c))])  # the support point linspace(-2, 2) in the ordered space
    vars_ = [Var("z", "z", n_groups), Var("sigma_a_log__", "sigma_a", 1, "log"), Var("beta", "beta", n_features),
             Var("cutpoints_ordered__", "cutpoints", K - 1, "ordered", initial=z0)]
    priors = [Prior("normal", "z", (0.0, 1.0)), Prior("halfnormal", "sigma_a_log__", (1.0,)), Prior("normal", "beta", (0.0, 1.0)),
              Prior("normal", "cutpoints_ordered__", (Linear([Term([], coef=mu_c)]), 5.0))]
    s = None
    if link == "probit":
        s = 1.0
        if sigma == "var":
            vars_.append(Var("sigma_log__", "sigma", 1, "log"))
            priors.append(Prior("halfnormal", "sigma_log__", (1.0,)))
            s = Ref("sigma_log__")
    terms = [Term([("sigma_a_log__", None), ("z", g)]), Term([("beta", None)], coef=X)]
    return ModelIR(name=f"ordinal_{link}", vars=vars_, priors=priors,
                   likelihoods=[Likelihood(f"ordered_{link}", y, terms, sigma=s, cutpoints=Ref("cutpoints_ordered__"))])


def zero_inflated_ir(dist: str = "zero_inflated_poisson", psi: str = "const", n_obs: int = 300, n_groups: int = 6,
                     n_features: int = 2, seed: int = 59) -> ModelIR:
    """A zero-inflated or hurdle regression (``dist`` in ZI_LIKS) on simulated data with real excess zeros:
    b0 ~ Normal(0, 2), z_g ~ Normal(0, 1) and sigma_a ~ HalfNormal(1) (non-centred group intercepts sigma_a z[g_i]),
    beta ~ Normal(0, 1)^F as a design term, eta_i = b0 + sigma_a z[g_i] + x_i . beta; the family's alpha ~ Exponential(1)
    (NegativeBinomial) or HalfNormal(2) (Gamma), and trials 0..11 per observation (Binomial).  psi: "const" (0.65),
    "var" (psi ~ Beta(2, 2) on interval(0, 1)) or "logit" (logit psi_i = g0 + w_i . gamma with g0 ~ Normal(0, 1.5) and
    gamma ~ Normal(0, 1)^2 as a design term)."""
    if dist not in ZI_FAMILY:
        raise ValueError(f"dist must be one of {ZI_LIKS}")
    if psi not in ("const", "var", "logit"):
        raise ValueError("psi must be 'const', 'var' or 'logit'")
    rng = np.random.default_rng(seed)
    fam = ZI_FAMILY[dist]
    g = rng.integers(0, n_groups, n_obs).astype(np.int32)
    X = rng.standard_normal((n_obs, n_features))
    Zp = rng.standard_normal((n_obs, 2))
    eta = 0.8 + rng.normal(0.0, 0.5, n_groups)[g] + X @ rng.normal(0.0, 0.4, n_features)
    psi_true = {"const": np.full(n_obs, 0.65), "var": np.full(n_obs, 0.6),
                "logit": 1.0 / (1.0 + np.exp(-(0.4 + Zp @ np.array([0.8, -0.6]))))}[psi]
    mu, a_true = np.exp(eta), 2.0
    trials = rng.integers(0, 12, n_obs).astype(np.float64) if fam == "binomial_logit" else None

    def draw(i):
        if fam == "poisson_log":
            return rng.poisson(mu[i])
        if fam == "binomial_logit":
            return rng.binomial(int(trials[i]), 1.0 / (1.0 + np.exp(-eta[i])))
        if fam == "negative_binomial_log":
            return rng.negative_binomial(a_true, a_true / (mu[i] + a_true))
        return rng.gamma(a_true, mu[i] / a_true)

    y = np.zeros(n_obs)
    for i in range(n_obs):
        if rng.random() < psi_true[i]:
            v = draw(i)
            while dist.startswith("hurdle") and fam != "gamma_log" and v == 0:  # Truncated(f, lower=1)
                v = draw(i)
            y[i] = v
    vars_ = [Var("b0", "b0", 1), Var("z", "z", n_groups), Var("sigma_a_log__", "sigma_a", 1, "log"),
             Var("beta", "beta", n_features)]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "z", (0.0, 1.0)), Prior("halfnormal", "sigma_a_log__", (1.0,)),
              Prior("normal", "beta", (0.0, 1.0))]
    alpha = None
    if fam in DISPERSION_LIKS:
        vars_.append(Var("alpha_log__", "alpha", 1, "log"))
        priors.append(Prior("exponential" if fam == "negative_binomial_log" else "halfnormal", "alpha_log__",
                            (1.0,) if fam == "negative_binomial_log" else (2.0,)))
        alpha = Ref("alpha_log__")
    if psi == "const":
        p = 0.65
    elif psi == "var":
        vars_.append(Var("psi_logodds__", "psi", 1, "interval", bounds=(0.0, 1.0)))
        priors.append(Prior("beta", "psi_logodds__", (2.0, 2.0)))
        p = Ref("psi_logodds__")
    else:
        vars_ += [Var("g0", "g0", 1), Var("gamma", "gamma", 2)]
        priors += [Prior("normal", "g0", (0.0, 1.5)), Prior("normal", "gamma", (0.0, 1.0))]
        p = Linear([Term([("g0", None)]), Term([("gamma", None)], coef=Zp)])
    terms = [Term([("b0", None)]), Term([("sigma_a_log__", None), ("z", g)]), Term([("beta", None)], coef=X)]
    return ModelIR(name=f"{dist}_{psi}", vars=vars_, priors=priors,
                   likelihoods=[Likelihood(dist, y, terms, alpha=alpha, trials=trials, psi=p)])


def survival_regression_ir(dist: str = "weibull", observe: str = "right_censored", alpha: float | None = None,
                           n_obs: int = 400, n_groups: int = 8, n_features: int = 3, seed: int = 61) -> ModelIR:
    """Survival regression on simulated event times, accelerated-failure-time style: eta_i = b0 + sigma_a z[g_i] + x_i . beta
    with b0 ~ Normal(0, 2), z_g ~ Normal(0, 1) and sigma_a ~ HalfNormal(1) (a non-centred group frailty), beta ~ Normal(0,
    1)^F as a design term, and T_i ~ Weibull(alpha, beta = exp(eta_i)) (``dist="weibull"``), Exponential(scale =
    exp(eta_i)), the Weibull with alpha = 1 (``"exponential"``), or LogNormal(eta_i, sigma) (``"lognormal"``).  The shape
    alpha ~ HalfNormal(2), the LogNormal's sigma ~ HalfNormal(1), or the constant ``alpha`` for either.
    observe: "plain" records every T_i; "right_censored" records y_i = min(T_i, c_i) at per-observation follow-up times
    c_i, which end about 30 % of the observations before their event; "entry_truncated" records subjects only if they are
    still event-free at their own entry time e_i (delayed entry; e_i = 0 for a third of them), i.e. T_i truncated to
    (e_i, inf)."""
    if dist not in ("weibull", "exponential", "lognormal"):
        raise ValueError("dist must be 'weibull', 'exponential' or 'lognormal'")
    if observe not in ("plain", "right_censored", "entry_truncated"):
        raise ValueError("observe must be 'plain', 'right_censored' or 'entry_truncated'")
    if dist == "exponential" and alpha is not None:
        raise ValueError("the exponential's shape is 1: leave alpha None")
    rng = np.random.default_rng(seed)
    g = rng.integers(0, n_groups, n_obs).astype(np.int32)
    X = rng.standard_normal((n_obs, n_features))
    eta = 1.0 + rng.normal(0.0, 0.4, n_groups)[g] + X @ rng.normal(0.0, 0.4, n_features)
    shape = 1.0 if dist == "exponential" else (1.5 if alpha is None else float(alpha))  # the Weibull's alpha
    scale = 0.8 if alpha is None else float(alpha)  # the LogNormal's sigma

    def draw(i):
        if dist == "lognormal":
            return float(np.exp(eta[i] + scale * rng.standard_normal()))
        return float(np.exp(eta[i]) * rng.exponential() ** (1.0 / shape))

    lower = upper = None
    entry = np.where(rng.random(n_obs) < 1 / 3, 0.0, np.exp(eta) * rng.uniform(0.05, 1.0, n_obs))
    y = np.empty(n_obs)
    for i in range(n_obs):
        y[i] = draw(i)
        while observe == "entry_truncated" and not y[i] > entry[i]:  # rejection: T_i given T_i > e_i
            y[i] = draw(i)
    if observe == "right_censored":
        u = np.exp(eta) * rng.uniform(0.5, 3.0, n_obs)
        upper = u * np.quantile(y / u, 0.7)  # 30 % of the T_i lie past their follow-up time
        y = np.minimum(y, upper)
    elif observe == "entry_truncated":
        lower = entry
    vars_ = [Var("b0", "b0", 1), Var("z", "z", n_groups), Var("sigma_a_log__", "sigma_a", 1, "log"),
             Var("beta", "beta", n_features)]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "z", (0.0, 1.0)), Prior("halfnormal", "sigma_a_log__", (1.0,)),
              Prior("normal", "beta", (0.0, 1.0))]
    par = 1.0 if dist == "exponential" else alpha
    if par is None:
        name = "sigma" if dist == "lognormal" else "alpha"
        vars_.append(Var(f"{name}_log__", name, 1, "log"))
        priors.append(Prior("halfnormal", f"{name}_log__", (1.0 if dist == "lognormal" else 2.0,)))
        par = Ref(f"{name}_log__")
    base = "lognormal" if dist == "lognormal" else "weibull_log"
    lik = {"plain": base, "right_censored": f"censored_{base}", "entry_truncated": f"truncated_{base}"}[observe]
    terms = [Term([("b0", None)]), Term([("sigma_a_log__", None), ("z", g)]), Term([("beta", None)], coef=X)]
    slot = dict(sigma=par) if dist == "lognormal" else dict(alpha=par)
    return ModelIR(name=f"survival_{dist}_{observe}", vars=vars_, priors=priors,
                   likelihoods=[Likelihood(lik, y, terms, lower=lower, upper=upper, **slot)])


def mixture_ir(dist: str = "normal", K: int = 3, weights: str = "dirichlet", covariates: int = 0, n_obs: int = 300,
               seed: int = 67) -> ModelIR:
    """A finite mixture on simulated data, the NormalMixture example of mixture.py:529-546: w ~ Dirichlet(ones(K)) on the
    simplex (``weights="dirichlet"``) or the constant weights of the simulation (``"const"``), and
    ``dist="normal"``: mu ~ Normal(0, 10)^K with the ordered transform, sigma ~ HalfNormal(2)^K,
    y_i ~ NormalMixture(w, eta_i + mu, sigma);  ``dist="poisson"``: lam ~ Normal(0, 20)^K with the ordered_positive
    transform (a HalfNormal(20) up to its constant), y_i ~ Mixture(w, Poisson(lam exp(eta_i))).  Ordered locations / rates keep the posterior free of label
    switching.  ``covariates`` > 0 adds beta ~ Normal(0, 1)^F as a design term, eta_i = x_i . beta (a shared shift, or a
    shared rate multiplier); with none, eta = 0.  A large K or a design term makes n > 256 (a chain per CTA)."""
    if dist not in ("normal", "poisson"):
        raise ValueError("dist must be 'normal' or 'poisson'")
    if weights not in ("dirichlet", "const"):
        raise ValueError("weights must be 'dirichlet' or 'const'")
    rng = np.random.default_rng(seed)
    w_true = np.linspace(1.0, 2.0, K)
    w_true /= w_true.sum()
    X = rng.standard_normal((n_obs, covariates))
    eta = X @ rng.normal(0.0, 0.3, covariates) if covariates else np.zeros(n_obs)
    z = rng.choice(K, n_obs, p=w_true)
    vars_, priors = [], []
    if weights == "dirichlet":
        vars_.append(Var("w_simplex__", "w", K - 1, "simplex"))
        priors.append(Prior("dirichlet", "w_simplex__", (np.ones(K),)))
        wt = Ref("w_simplex__")
    else:
        wt = w_true
    if dist == "normal":
        mu_true = np.linspace(-3.0 * (K - 1), 3.0 * (K - 1), K) / max(K - 1, 1)
        y = eta + mu_true[z] + 0.8 * rng.standard_normal(n_obs)
        z0 = np.concatenate([[mu_true[0]], np.log(np.diff(mu_true))])
        vars_ += [Var("mu_ordered__", "mu", K, "ordered", initial=z0), Var("sigma_log__", "sigma", K, "log")]
        priors += [Prior("normal", "mu_ordered__", (0.0, 10.0)), Prior("halfnormal", "sigma_log__", (2.0,))]
        comp, sg, lik = Ref("mu_ordered__"), Ref("sigma_log__"), "normal_mixture"
    else:
        lam_true = 2.0 * 3.0 ** np.arange(K) / 3.0 ** ((K - 1) / 2)
        y = rng.poisson(lam_true[z] * np.exp(eta)).astype(np.float64)
        z0 = np.concatenate([[np.log(lam_true[0])], np.log(np.diff(lam_true))])
        vars_.append(Var("lam_ordered__", "lam", K, "ordered_positive", initial=z0))
        priors.append(Prior("normal", "lam_ordered__", (0.0, 20.0)))
        comp, sg, lik = Ref("lam_ordered__"), None, "poisson_mixture"
    terms = []
    if covariates:
        vars_.append(Var("beta", "beta", covariates))
        priors.append(Prior("normal", "beta", (0.0, 1.0)))
        terms = [Term([("beta", None)], coef=X)]
    return ModelIR(name=f"{dist}_mixture_{K}_{weights}", vars=vars_, priors=priors,
                   likelihoods=[Likelihood(lik, y, terms, sigma=sg, weights=wt, components=comp)])


def beta_regression_ir(dist: str = "beta", phi: str = "var", n_obs: int = 400, n_groups: int = 8, n_features: int = 2,
                       seed: int = 71) -> ModelIR:
    """Beta regression on simulated data: eta_i = b0 + sigma_a z[g_i] + x_i . beta with b0 ~ Normal(0, 1.5), z_g ~ Normal(0,
    1) and sigma_a ~ HalfNormal(1) (non-centred group intercepts), beta ~ Normal(0, 1)^F as a design term, mu_i =
    sigmoid(eta_i), and ``dist="beta"``: y_i ~ Beta(mu_i, nu = phi), the proportions PyMC writes as
    ``pm.Beta("y", mu=pm.math.invlogit(eta), nu=phi)``; ``"beta_binomial"``: y_i ~ BetaBinomial(n_i, phi mu_i, phi (1 -
    mu_i)) with per-observation trials n_i from 5 to 60, whose spread is visibly wider than the Binomial's (phi = 4).
    ``phi="var"``: phi ~ Gamma(2, 0.1) under a log transform; ``"const"``: phi is the simulation's value."""
    if dist not in ("beta", "beta_binomial"):
        raise ValueError("dist must be 'beta' or 'beta_binomial'")
    if phi not in ("var", "const"):
        raise ValueError("phi must be 'var' or 'const'")
    rng = np.random.default_rng(seed)
    g = rng.integers(0, n_groups, n_obs).astype(np.int32)
    X = rng.standard_normal((n_obs, n_features))
    eta = -0.3 + rng.normal(0.0, 0.5, n_groups)[g] + X @ rng.normal(0.0, 0.5, n_features)
    mu = 1.0 / (1.0 + np.exp(-eta))
    phi_true = 15.0 if dist == "beta" else 4.0
    p = rng.beta(mu * phi_true, (1.0 - mu) * phi_true)
    trials = None
    if dist == "beta":
        y = np.clip(p, 1e-12, 1.0 - 1e-12)
    else:
        trials = rng.integers(5, 61, n_obs).astype(np.float64)
        y = rng.binomial(trials.astype(np.int64), p).astype(np.float64)
    vars_ = [Var("b0", "b0", 1), Var("z", "z", n_groups), Var("sigma_a_log__", "sigma_a", 1, "log"),
             Var("beta", "beta", n_features)]
    priors = [Prior("normal", "b0", (0.0, 1.5)), Prior("normal", "z", (0.0, 1.0)), Prior("halfnormal", "sigma_a_log__", (1.0,)),
              Prior("normal", "beta", (0.0, 1.0))]
    par = phi_true
    if phi == "var":
        vars_.append(Var("phi_log__", "phi", 1, "log", initial=np.log(phi_true)))
        priors.append(Prior("gamma", "phi_log__", (2.0, 0.1)))
        par = Ref("phi_log__")
    terms = [Term([("b0", None)]), Term([("sigma_a_log__", None), ("z", g)]), Term([("beta", None)], coef=X)]
    lik = "beta_logit" if dist == "beta" else "beta_binomial_logit"
    return ModelIR(name=f"{dist}_{phi}", vars=vars_, priors=priors,
                   likelihoods=[Likelihood(lik, y, terms, trials=trials, phi=par)])


def hsgp_regression_ir(cov: str = "expquad", dims: int = 1, ls: str = "var", amplitude: str = "var", dist: str = "normal",
                       n_obs: int = 300, m: int | None = None, c: float = 1.5, additive: bool = False, covariates: int = 0,
                       seed: int = 83) -> ModelIR:
    """A GP regression through the non-centred HSGP on simulated data, as ``pm.gp.HSGP(m, c, cov_func=eta**2 * cov).prior``
    writes it: f = Phi (z * s(ell, eta)) with z ~ Normal(0, 1)^M, ell ~ InverseGamma(4, 4 ell_0) (ARD: one per input
    dimension) and eta ~ HalfNormal(1), both under log transforms.  X is uniform on [0, 10]^dims and the data come from a
    smooth known f.  ``ls`` / ``amplitude`` = "const" fixes them at the simulation's values (a plain design term).
    ``additive``: a second HSGP term with its own shorter lengthscale and amplitude; ``covariates`` = F > 0: an intercept
    b0 ~ Normal(0, 2) and a design term X_c beta_c.  ``dist``: "normal" (sigma ~ HalfNormal(1)), "poisson" (log link) or
    "bernoulli" (logit link).  ``m`` basis functions per dimension (default 24 in 1-D, 12 per dimension in 2-D).  The GP's
    values are recorded as the Deterministic ``f``."""
    if cov not in COV_FUNCS:
        raise ValueError(SPEC_COV)
    if dist not in ("normal", "poisson", "bernoulli") or ls not in ("var", "const") or amplitude not in ("var", "const"):
        raise ValueError("dist must be normal, poisson or bernoulli; ls and amplitude 'var' or 'const'")
    m = m or (24 if dims == 1 else 12)
    rng = np.random.default_rng(seed)
    X = rng.uniform(0.0, 10.0, (n_obs, dims))
    truth = np.sin(X[:, 0]) + (0.5 * np.cos(0.6 * X[:, 1]) if dims > 1 else 0.0)
    vars_, priors, terms, gp_terms = [], [], [], []

    def gp(tag, ell0, eta0, mm):
        Phi, omega, _, _ = hsgp_basis(X, [mm] * dims, c=c)
        M = Phi.shape[1]
        z = f"{tag}_hsgp_coeffs"
        vars_.append(Var(z, z, M))
        priors.append(Prior("normal", z, (0.0, 1.0)))
        lsv, av = np.full(dims, ell0) if dims > 1 else ell0, eta0
        if ls == "var":
            vars_.append(Var(f"ell_{tag}_log__", f"ell_{tag}", dims, "log", initial=np.log(ell0)))
            priors.append(Prior("inversegamma", f"ell_{tag}_log__", (4.0, 4.0 * ell0)))
            lsv = Ref(f"ell_{tag}_log__")
        if amplitude == "var":
            vars_.append(Var(f"eta_{tag}_log__", f"eta_{tag}", 1, "log", initial=np.log(eta0)))
            priors.append(Prior("halfnormal", f"eta_{tag}_log__", (1.0,)))
            av = Ref(f"eta_{tag}_log__")
        t = Term([(z, None)], coef=Phi, spectral=Spectral(cov, omega, lsv, av))
        terms.append(t)
        gp_terms.append(t)

    gp("f", 2.0, 1.0, m)
    if additive:
        truth = truth + 0.3 * np.sin(3.0 * X[:, 0])
        gp("g", 0.4, 0.3, m)
    eta = truth
    if covariates:
        Xc = rng.standard_normal((n_obs, covariates))
        eta = eta + 0.3 + Xc @ rng.normal(0.0, 0.5, covariates)
        vars_ += [Var("b0", "b0", 1), Var("beta", "beta", covariates)]
        priors += [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "beta", (0.0, 1.0))]
        terms += [Term([("b0", None)]), Term([("beta", None)], coef=Xc)]
    if dist == "normal":
        y = eta + rng.normal(0.0, 0.3, n_obs)
        vars_.append(Var("sigma_log__", "sigma", 1, "log", initial=np.log(0.3)))
        priors.append(Prior("halfnormal", "sigma_log__", (1.0,)))
        lik = Likelihood("normal", y, terms, sigma=Ref("sigma_log__"))
    elif dist == "poisson":
        lik = Likelihood("poisson_log", rng.poisson(np.exp(0.5 + eta)).astype(np.float64), terms)
    else:
        lik = Likelihood("bernoulli_logit", (rng.random(n_obs) < 1.0 / (1.0 + np.exp(-2.0 * eta))).astype(np.float64), terms)
    return ModelIR(name=f"hsgp_{cov}_{dims}d_{dist}", vars=vars_, priors=priors, likelihoods=[lik],
                   deterministics=[Deterministic("f", n_obs, gp_terms)])


# ------------------------------------------------------------------------------------------------------------------------
# lowering: ModelIR -> flat arrays of the C ABI (include/b200nuts.h: b200_ir)
# ------------------------------------------------------------------------------------------------------------------------
@dataclass
class LoweredIR:
    """Integer and double tables + data arrays; ``_lib`` turns them into ctypes structures."""

    n: int
    vars: np.ndarray        # [n_vars] (offset, size, transform) int32 x3 ; bounds in var_bounds
    var_bounds: np.ndarray  # [n_vars][2]
    priors: list            # [(dist, var, [(kind, value, ref_offset)] * 3)]
    liks: list              # [dict(dist, N, y, terms=[dict(coef, factors=[(offset, size, idx)])], sigma_kind, sigma_value, sigma_ref, sigma_obs, nu, y_var)]
                            # a design term's dict also has n_cols = K, with coef = X [N][K]
                            # censored_normal / truncated_normal and the censored_ / truncated_ survival likelihoods:
                            # y is the [3][N] block (y, lower, upper); the Weibull's alpha is the sigma slot
                            # ordered_logistic / ordered_probit: nu = K, and cut = the cutpoint term (a term dict)
                            # zero-inflated / hurdle: nu = 0 or m, and psi = the psi block (a list of term dicts)
                            # normal_mixture / poisson_mixture: nu = K, and mix = the weights, component (and sigma)
                            # blocks (term dicts)
                            # beta_logit / beta_binomial_logit: phi is the sigma slot; beta_binomial_logit's y is the
                            # [2][N] block (y, trials)
                            # y_var 0: y is observed data; v + 1: a latent factor, y is None and its values are variable v's
    ar1: list               # [(var, phi(kind, value, ref), sigma(kind, value, ref), init_sigma)]


def _param(ir: ModelIR, a, off):
    if isinstance(a, Ref):
        v = ir.var(a.var)
        return (1, 0.0, off[v.name])
    return (0, float(a), -1)


def _lower_terms(ir: ModelIR, terms: list, N: int, off: dict) -> list:
    out = []
    for t in terms:
        if t.spectral is not None:
            out.append(_lower_spectral(ir, t, off))
            continue
        if is_design(t):  # one ABI design term: coef = X row-major, n_cols = K
            v = ir.var(t.factors[0][0])
            out.append(dict(coef=np.ascontiguousarray(t.coef, dtype=np.float64), factors=[(off[v.name], v.size, None)],
                            n_cols=v.size))
            continue
        coef = None
        scale = 1.0
        if t.coef is not None:
            if np.ndim(t.coef) == 0:
                scale = float(t.coef)
            else:
                coef = np.ascontiguousarray(t.coef, dtype=np.float64)
        if scale != 1.0:
            coef = np.full(N, scale) if coef is None else coef * scale
        fs = []
        for vn, idx in t.factors:
            v = ir.var(vn)
            fs.append((off[v.name], v.size, None if idx is None else np.ascontiguousarray(idx, dtype=np.int32)))
        out.append(dict(coef=coef, factors=fs))
    return out


def _lower_spectral(ir: ModelIR, t, off: dict) -> dict:
    """A spectral term: with constant ls and amplitude, the design term X = Phi diag(s); else the ABI's spectral term,
    coef = Phi followed by the block (cov, D, amplitude, ls_1 .. ls_D, omega), factors z, amplitude and ls, where a size
    0 factor stands for the constants in the block (include/b200nuts.h)."""
    sp = t.spectral
    v = ir.var(t.factors[0][0])
    Phi = np.asarray(t.coef, dtype=np.float64)
    om = np.asarray(sp.omega, dtype=np.float64)
    M, D = om.shape
    if not isinstance(sp.ls, Ref) and not isinstance(sp.amplitude, Ref):
        s = np.exp(spectral_log_scale(sp.cov, om, np.broadcast_to(np.asarray(sp.ls, dtype=np.float64).reshape(-1), (D,)),
                                      float(sp.amplitude)))
        return dict(coef=np.ascontiguousarray(Phi * s[None, :]), factors=[(off[v.name], M, None)], n_cols=M)
    amp = (off[ir.var(sp.amplitude.var).name], 1, None) if isinstance(sp.amplitude, Ref) else (0, 0, None)
    ls = (off[ir.var(sp.ls.var).name], ir.var(sp.ls.var).size, None) if isinstance(sp.ls, Ref) else (0, 0, None)
    a_c = 0.0 if isinstance(sp.amplitude, Ref) else float(sp.amplitude)
    ls_c = np.zeros(D) if isinstance(sp.ls, Ref) else np.broadcast_to(np.asarray(sp.ls, dtype=np.float64).reshape(-1), (D,))
    blk = np.concatenate([[float(COV_FUNCS[sp.cov]), float(D), a_c], ls_c, om.ravel()])
    return dict(coef=np.ascontiguousarray(np.concatenate([Phi.ravel(), blk])), factors=[(off[v.name], M, None), amp, ls],
                n_cols=M)


def _lower_slot(ir: ModelIR, par, off: dict) -> dict:
    """A factor's parameter slot: none, a constant, a scalar variable or one constant per element."""
    sk, sv, sr, so = SIGMA_NONE, 0.0, -1, None
    if isinstance(par, Ref):
        sk, sr = SIGMA_REF, off[ir.var(par.var).name]
    elif par is not None and np.ndim(par) == 1:
        sk, so = SIGMA_OBS, np.ascontiguousarray(par, dtype=np.float64)
    elif par is not None:
        sk, sv = SIGMA_CONST, float(par)
    return dict(sigma_kind=sk, sigma_value=sv, sigma_ref=sr, sigma_obs=so)


def lower(ir: ModelIR) -> LoweredIR:
    ir.validate()
    off = ir.offsets()
    nv = len(ir.vars)
    vars_ = np.zeros((nv, 3), dtype=np.int32)
    bounds = np.zeros((nv, 2))
    index = {}
    for k, v in enumerate(ir.vars):
        vars_[k] = (off[v.name], v.size, TRANSFORMS[v.transform])
        if v.bounds:
            bounds[k] = v.bounds
        index[v.name] = k
    priors, latent = [], []
    for p in ir.priors:
        if is_latent(p):
            latent.append(p)
            continue
        if p.dist == "dirichlet":  # its one concentration (validate: one constant or K equal ones)
            pars = [(0, float(np.ravel(p.params[0])[0]), -1)] + [(0, 0.0, -1)] * 2
            priors.append((PRIOR_DISTS[p.dist][0], index[ir.var(p.var).name], pars))
            continue
        pars = [_param(ir, a, off) for a in p.params] + [(0, 0.0, -1)] * (3 - len(p.params))
        priors.append((PRIOR_DISTS[p.dist][0], index[ir.var(p.var).name], pars))
    liks = []
    for L in ir.likelihoods:
        # the likelihood's one parameter slot: sigma, or the trials / alpha of the count and positive families
        fam = ZI_FAMILY.get(L.dist, L.dist)
        par = L.trials if fam == "binomial_logit" else (L.alpha if fam in DISPERSION_LIKS + WEIBULL_LIKS else L.sigma)
        if L.dist in MIXTURE_LIKS:
            par = None  # sigma is a block
        if L.dist in BETA_LIKS:
            par = L.phi
        y = np.ascontiguousarray(L.y, dtype=np.float64)
        if L.dist == "beta_binomial_logit":  # the [2][N] block: y, trials
            y = np.ascontiguousarray(np.stack([y, np.broadcast_to(np.asarray(L.trials, dtype=np.float64), y.shape)]))
        if L.dist in BOUNDED_LIKS + SURVIVAL_BOUNDED:  # the [3][N] block: y, lower, upper
            y = np.ascontiguousarray(np.stack([y, *L.bounds()]))
        extra = {}
        if L.dist in ORDINAL_LIKS:  # nu = K; the cutpoint term goes one past the predictor's terms
            c = L.cutpoints
            extra = dict(nu=float(L.n_categories(ir)),
                         cut=dict(coef=None, factors=[(off[ir.var(c.var).name], ir.var(c.var).size, None)])
                         if isinstance(c, Ref) else dict(coef=np.ascontiguousarray(c, dtype=np.float64), factors=[]))
        if L.dist in MIXTURE_LIKS:  # nu = K; the weights, component and (normal) sigma blocks one past the predictor's terms
            K = L.n_components(ir)

            def block(a, n):
                if isinstance(a, Ref):
                    v = ir.var(a.var)
                    return dict(coef=None, factors=[(off[v.name], v.size, None)])
                return dict(coef=np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=np.float64), (n,))), factors=[])

            mix = [block(L.weights, K), block(L.components, K)] + ([block(L.sigma, K)] if L.dist == "normal_mixture" else [])
            extra = dict(nu=float(K), mix=mix)
        if L.dist in ZI_LIKS:  # the psi block goes one past the predictor's terms; nu = 0 (psi) or its number of terms
            psi = L.psi
            if isinstance(psi, Linear):
                extra = dict(nu=float(len(psi.terms)), psi=_lower_terms(ir, psi.terms, len(L.y), off))
            elif isinstance(psi, Ref):
                extra = dict(nu=0.0, psi=[dict(coef=None, factors=[(off[ir.var(psi.var).name], 1, None)])])
            else:
                extra = dict(nu=0.0, psi=[dict(coef=np.array([float(psi)]), factors=[])])
        liks.append(dict(dict(dist=LIK_DISTS[L.dist], N=len(L.y), y=y,
                              terms=_lower_terms(ir, L.terms, len(L.y), off), nu=float(L.nu), y_var=0,
                              **_lower_slot(ir, par, off)), **extra))
    # latent factors after the observed likelihoods, so that observed likelihood i keeps index i
    for p in latent:
        v = ir.var(p.var)
        loc, scale = LINEAR_PRIORS[p.dist]
        mu = p.params[loc]
        terms = mu.terms if isinstance(mu, Linear) else [Term([(mu.var, None)]) if isinstance(mu, Ref) else Term([], coef=float(mu))]
        liks.append(dict(dist=LIK_DISTS[p.dist], N=v.size, y=None, terms=_lower_terms(ir, terms, v.size, off),
                         nu=float(p.params[0]) if p.dist == "studentt" else 0.0, y_var=index[v.name] + 1,
                         **_lower_slot(ir, p.params[scale], off)))
    ar1 =[(index[ir.var(a.var).name], _param(ir, a.phi, off), _param(ir, a.sigma, off), float(a.init_sigma)) for a in ir.ar1]
    return LoweredIR(ir.n, vars_, bounds, priors, liks, ar1)


def _column_of(t, N: int, ir: ModelIR):
    """(variable name, k) when term t is column k of a design matrix written out: one factor on a vector variable of size
    K >= 2, gathered at the constant index k, times a 1-D coefficient of length N, a scalar or nothing; else None."""
    if len(t.factors) != 1 or t.factors[0][1] is None:
        return None
    vn, idx = t.factors[0]
    v = ir.var(vn)
    idx = np.asarray(idx)
    if v.size < 2 or idx.shape != (N,) or N == 0:
        return None
    k = int(idx[0])
    if not (0 <= k < v.size and np.all(idx == k)):
        return None
    if t.coef is not None and not (np.ndim(t.coef) == 0 or (np.ndim(t.coef) == 1 and len(t.coef) == N)):
        return None
    return v.name, k


def fuse_design_columns(model: ModelIR) -> ModelIR:
    """A copy of ``model`` in which, per likelihood and per ``Linear`` prior location, each complete run of column terms --
    one term per column k = 0..K-1 of the same vector variable of size K, as ``from_pymc`` lowers ``pm.math.dot(X, beta)``
    -- is one design term with X[:, k] = the column's coefficient, placed where the run's first term was.  Partial or
    duplicated runs, indexed group effects, multi-factor terms and Deterministics stay as written; ``model`` itself is
    not changed.  The terms of a likelihood's logit(psi) are fused the same way."""
    out = copy.deepcopy(model)
    for L in out.likelihoods:
        L.terms = _fuse_terms(out, L.terms, len(L.y))
        if isinstance(L.psi, Linear):  # logit(psi) of a zero-inflated / hurdle likelihood
            L.psi = Linear(_fuse_terms(out, L.psi.terms, len(L.y)))
    for p in out.priors:
        p.params = tuple(Linear(_fuse_terms(out, a.terms, out.var(p.var).size)) if isinstance(a, Linear) else a
                         for a in p.params)
    return out


def _fuse_terms(model: ModelIR, terms: list, N: int) -> list:
    runs = {}  # variable -> [(term position, k)]
    for j, t in enumerate(terms):
        ck = _column_of(t, N, model)
        if ck is not None:
            runs.setdefault(ck[0], []).append((j, ck[1]))
    fused, drop = {}, set()
    for vn, cols in runs.items():
        K = model.var(vn).size
        if sorted(k for _, k in cols) != list(range(K)):
            continue
        X = np.empty((N, K))
        for j, k in cols:
            c = terms[j].coef
            X[:, k] = 1.0 if c is None else np.asarray(c, dtype=np.float64)
        first = min(j for j, _ in cols)
        fused[first] = Term([(vn, None)], coef=X)
        drop.update(j for j, _ in cols)
    if not fused:
        return terms
    return [fused[j] if j in fused else t for j, t in enumerate(terms) if j in fused or j not in drop]


# ------------------------------------------------------------------------------------------------------------------------
# pattern -> hand-specialised kernel (fast paths behind the IR)
# ------------------------------------------------------------------------------------------------------------------------
def specialise(ir: ModelIR, extended: bool = False):
    """Return a ``models.ModelSpec`` of a hand-written kernel when the IR is one of the recognised shapes, else None.

    Recognised: the non-centred varying-intercept/varying-slope Normal regression of benchmarks.py:34-45 (Radon; any data),
    non-centred Eight Schools (any J), the AR(1) stochastic-volatility model of BASELINE config 4 (any T) and the logistic GLM
    of config 3 (beta ~ Normal(0, 1), up to 128 features: the fused design-matrix kernels, fp64 DMMA or wgmma) -- these two
    only with ``extended=True`` (``CompiledModel(ir, specialise="all")``): the routes were added after the round's last GPU run
    and are checked on the CPU only (the specialised spec has the IR's density, tests/test_ir.py), so the default keeps such
    models on the generic function.  Everything else runs on the generic IR device function."""
    from . import models

    def const(p, k, want=None):
        return not isinstance(p.params[k], Ref) and (want is None or float(p.params[k]) == want)

    if any(t.spectral is not None for L in ir.likelihoods for t in L.terms):
        return None
    pri = {ir.var(p.var).name: p for p in ir.priors}
    if len(pri) != len(ir.priors) or len(ir.likelihoods) != 1 or ir.likelihoods[0].dist in ZI_LIKS + MIXTURE_LIKS + BETA_LIKS:
        return None
    if any(isinstance(a, Linear) or (not isinstance(a, Ref) and np.ndim(a) > 0) for p in ir.priors for a in p.params):
        return None
    L = ir.likelihoods[0]
    names = [v.name for v in ir.vars]
    tr = [v.transform for v in ir.vars]
    sizes = [v.size for v in ir.vars]

    def plain(t, vn):  # the term is exactly the variable: no coefficient, no gather index
        return t.coef is None and len(t.factors) == 1 and t.factors[0][0] == vn and t.factors[0][1] is None

    # ---- stochastic volatility (BASELINE config 4): [mu, phi (interval -1, 1), log sigma, h[T]] ------------------------
    if extended and len(ir.ar1) == 1 and L.dist == "normal_logvar":
        A = ir.ar1[0]
        if not (len(names) == 4 and tr == [None, "interval", "log", None] and sizes[:3] == [1, 1, 1] and sizes[3] == len(L.y)
                and tuple(ir.vars[1].bounds or ()) == (-1.0, 1.0) and len(pri) == 3 and L.sigma is None and len(L.terms) == 2):
            return None
        mu, phi, sg, h = names
        ok = (ir.var(A.var).name == h and isinstance(A.phi, Ref) and ir.var(A.phi.var).name == phi
              and isinstance(A.sigma, Ref) and ir.var(A.sigma.var).name == sg and float(A.init_sigma) == 1.0
              and plain(L.terms[0], mu) and plain(L.terms[1], h)
              and mu in pri and pri[mu].dist == "normal" and const(pri[mu], 0, 0.0) and const(pri[mu], 1, 5.0)
              and phi in pri and pri[phi].dist == "uniform" and const(pri[phi], 0, -1.0) and const(pri[phi], 1, 1.0)
              and sg in pri and pri[sg].dist == "exponential" and const(pri[sg], 0, 10.0))
        if not ok:
            return None
        spec = models.stochvol(T=4)  # layout donor; data and sizes replaced below
        T = len(L.y)
        spec.n = T + 3
        spec.vars, _ = models._layout([(v.name, v.rv_name, v.size, v.transform, v.bounds) for v in ir.vars])
        spec.data = {"y": np.asarray(L.y, dtype=np.float64)}
        spec.meta = {"T": T, "initial_point": ir.initial_point()}
        return spec
    if ir.ar1:
        return None
    # ---- logistic GLM (BASELINE config 3): beta ~ Normal(0, 1)^K, y ~ Bernoulli(logit_p = X beta), K <= 128 --------------
    if extended and L.dist == "bernoulli_logit":
        design = len(L.terms) == 1 and is_design(L.terms[0])  # X beta as one design term, or as one term per column
        if not (len(names) == 1 and tr == [None] and 1 <= sizes[0] <= 128 and (design or len(L.terms) == sizes[0])):
            return None
        beta, K, N = names[0], sizes[0], len(L.y)
        if not (beta in pri and pri[beta].dist == "normal" and const(pri[beta], 0, 0.0) and const(pri[beta], 1, 1.0)):
            return None
        if not np.all((np.asarray(L.y) == 0) | (np.asarray(L.y) == 1)):
            return None
        if design:
            t = L.terms[0]
            if ir.var(t.factors[0][0]).name != beta or np.shape(t.coef) != (N, K):
                return None
            X = np.array(t.coef, dtype=np.float64)
        else:
            X = np.empty((N, K))
            seen = set()
            for t in L.terms:
                if len(t.factors) != 1 or t.factors[0][0] != beta or t.factors[0][1] is None or np.ndim(t.coef) != 1 or len(t.coef) != N:
                    return None
                ix = np.asarray(t.factors[0][1])
                k = int(ix[0])
                if k in seen or not (0 <= k < K) or not np.all(ix == k):
                    return None
                seen.add(k)
                X[:, k] = t.coef
        spec = models.logistic(n_rows=4, n_features=2)  # layout donor
        spec.n = K
        spec.vars, _ = models._layout([(beta, ir.vars[0].rv_name, K, None, None)])
        spec.data = {"X": X, "y": np.asarray(L.y).astype(np.uint8)}
        spec.meta = {"n_rows": N, "initial_point": ir.initial_point()}
        return spec
    if L.dist != "normal":
        return None
    # ---- Eight Schools: [mu, log tau, theta_t[J]] ---------------------------------------------------------------
    if (len(names) == 3 and tr == [None, "log", None] and sizes[:2] == [1, 1] and sizes[2] == len(L.y)
            and np.ndim(L.sigma) == 1 and len(L.terms) == 2):
        mu, tau, th = names
        t0, t1 = L.terms
        ok = (t0.coef is None and [f[0] for f in t0.factors] == [mu]
              and t1.coef is None and sorted(f[0] for f in t1.factors) == sorted([tau, th])
              and all(f[1] is None for f in t0.factors + t1.factors)
              and pri[mu].dist == "normal" and const(pri[mu], 0, 0.0) and const(pri[mu], 1, 5.0)
              and pri[tau].dist == "halfcauchy" and const(pri[tau], 0, 5.0)
              and pri[th].dist == "normal" and const(pri[th], 0, 0.0) and const(pri[th], 1, 1.0))
        if ok:
            spec = models.eight_schools()
            spec.data = {"y": np.asarray(L.y, dtype=np.float64), "sigma": np.asarray(L.sigma, dtype=np.float64)}
            spec.n = len(L.y) + 2
            spec.vars, _ = models._layout([(mu, ir.vars[0].rv_name, 1, None, None), (tau, ir.vars[1].rv_name, 1, "log", None),
                                           (th, ir.vars[2].rv_name, len(L.y), None, None)])
            spec.meta = {"initial_point": ir.initial_point()}
            return spec
    # ---- Radon: [mu_a, log sigma_a, mu_b, log sigma_b, a[J], b[J], log eps] ----------------------------------------
    if len(names) == 7 and tr == [None, "log", None, "log", None, None, "log"] and sizes[4] == sizes[5] and \
            sizes[:4] == [1, 1, 1, 1] and sizes[6] == 1 and isinstance(L.sigma, Ref) and len(L.terms) == 4:
        mu_a, sa, mu_b, sb, a, b, eps = names
        if ir.var(L.sigma.var).name != eps:
            return None
        want = [({mu_a}, False), ({sa, a}, False), ({mu_b}, True), ({sb, b}, True)]
        idx, x = None, None
        for t, (vs, has_coef) in zip(L.terms, want):
            if {f[0] for f in t.factors} != vs or len(t.factors) != len(vs) or (t.coef is not None) != has_coef:
                return None
            for vn, ix in t.factors:
                if vn in (a, b):
                    if ix is None or (idx is not None and not np.array_equal(ix, idx)):
                        return None
                    idx = ix
                elif ix is not None:
                    return None
            if has_coef:
                if np.ndim(t.coef) != 1 or (x is not None and not np.array_equal(t.coef, x)):
                    return None
                x = t.coef
        ok = (pri[mu_a].dist == "normal" and const(pri[mu_a], 0, 0.0) and const(pri[mu_a], 1, 1.0e4)
              and pri[mu_b].dist == "normal" and const(pri[mu_b], 0, 0.0) and const(pri[mu_b], 1, 1.0e4)
              and all(pri[s].dist == "halfcauchy" and const(pri[s], 0, 5.0) for s in (sa, sb, eps))
              and all(pri[s].dist == "normal" and const(pri[s], 0, 0.0) and const(pri[s], 1, 1.0) for s in (a, b)))
        if ok:
            J = sizes[4]
            spec = models.radon(8, 2, 0)  # layout donor; data and sizes replaced below
            spec.n = 2 * J + 5
            spec.vars, _ = models._layout([(v.name, v.rv_name, v.size, v.transform, None) for v in ir.vars])
            spec.data = {"county_idx": np.asarray(idx, dtype=np.int32), "floor": np.asarray(x, dtype=np.float64),
                         "y": np.asarray(L.y, dtype=np.float64)}
            spec.meta = {"n_counties": J, "n_obs": len(L.y), "initial_point": ir.initial_point()}
            return spec
    return None
