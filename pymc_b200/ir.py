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
from dataclasses import dataclass, field

import numpy as np

# ids shared with include/b200nuts.h ------------------------------------------------------------------------------------
TRANSFORMS = {None: 0, "log": 1, "interval": 2}
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
}
DISPERSION_LIKS = ("negative_binomial_log", "gamma_log")  # their `alpha` is a constant or a Ref
# The support rule.  The device evaluates a density's formula wherever it is asked to, so every variable must be kept
# inside its prior's support by its transform, and every scale parameter must be positive:
POSITIVE_PRIORS = ("halfnormal", "halfcauchy", "exponential", "gamma", "lognormal")  # a log transform, or interval lo >= 0
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
    return v.transform == "log" or (v.transform == "interval" and v.bounds[0] >= 0.0)


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
class Term:
    """coef[i] * prod_f x_f[idx_f[i]].  A factor's idx is None for a scalar variable (broadcast) or for a vector variable of
    the likelihood's own length (elementwise).

    A design term has a 2-D coef X of shape [N][K] and exactly one factor, a variable of size K with no index:
    it adds sum_k X[i, k] * x[k], i.e. ``pm.math.dot(X, beta)``, evaluated on the device as one team-parallel term."""

    factors: list  # [(var_name, idx or None), ...]
    coef: np.ndarray | float | None = None


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
    alpha: float | Ref | None = None           # negative_binomial_log / gamma_log: dispersion (shape)
    trials: float | np.ndarray | None = None   # binomial_logit: number of trials, one for all or one per observation


@dataclass
class Deterministic:
    """``pm.Deterministic(name, expr)`` whose expression is a linear predictor of the CONSTRAINED variables (the same closed form as
    a likelihood's location): recorded in the posterior group like the reference's trace does (model/core.py:1956-2040,
    backends/base.py:184-191), evaluated on the host from the draws -- it never enters logp."""

    name: str
    size: int
    terms: list


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
        for p in self.priors:
            if p.dist not in PRIOR_DISTS:
                raise ValueError(f"prior {p.dist!r} is not in the closed set {sorted(PRIOR_DISTS)}")
            if len(p.params) != PRIOR_DISTS[p.dist][1]:
                raise ValueError(f"prior {p.dist} on {p.var}: expected {PRIOR_DISTS[p.dist][1]} parameters")
            v = self.var(p.var)
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
                    if p.dist in ("uniform", "gamma", "beta") or (p.dist == "studentt" and k == 0):
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
        for L in self.likelihoods:
            if L.dist not in LIK_DISTS:
                raise ValueError(f"likelihood {L.dist!r} is not in the closed set {sorted(LIK_DISTS)}")
            N = len(L.y)
            self._check_terms(L.terms, N, f"likelihood {L.name}", "the number of observations")
            if L.dist in ("normal", "studentt") and L.sigma is None:
                raise ValueError(f"{L.dist} likelihood needs sigma")
            if isinstance(L.sigma, Ref) and self.var(L.sigma.var).size != 1:
                raise ValueError("likelihood sigma must be a scalar variable")
            if L.dist in ("normal", "studentt"):
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
        for a in self.ar1:
            if self.var(a.var).size < 2:
                raise ValueError("AR1 needs at least two steps")
            for r in (a.phi, a.sigma):
                if isinstance(r, Ref) and self.var(r.var).size != 1:
                    raise ValueError("AR1 parameters must be scalar variables or constants")
            self._check_scale(a.sigma, f"AR1 on {a.var}: sigma")
            if not (np.isfinite(a.init_sigma) and a.init_sigma > 0):
                raise ValueError(f"AR1 on {a.var}: init_sigma must be > 0")

    def _check_terms(self, terms, N: int, where: str, length: str) -> None:
        """Terms of a predictor of length N (a likelihood's observations, or the elements of a prior's variable)."""
        for t in terms:
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
        if p.dist in POSITIVE_PRIORS and not _positive_support(v):
            raise ValueError(f"prior {p.dist} on {v.name}: the variable needs a log transform or an interval with lo >= 0 "
                             "(positive support)")
        if p.dist == "studentt" and not (np.isfinite(float(p.params[0])) and float(p.params[0]) > 0):
            raise ValueError(f"prior studentt on {v.name}: StudentT nu must be a positive constant")
        if p.dist in ("gamma", "beta") and not all(np.isfinite(float(a)) and float(a) > 0 for a in p.params):
            raise ValueError(f"prior {p.dist} on {v.name}: {p.dist.capitalize()} needs constant alpha, beta > 0")
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
        if L.dist == "binomial_logit":
            if L.trials is None or isinstance(L.trials, Ref):
                raise ValueError("binomial_logit: trials must be a constant scalar or a constant array")
            n = np.asarray(L.trials, dtype=np.float64)
            if n.ndim > 1 or (n.ndim == 1 and len(n) != len(y)):
                raise ValueError("binomial_logit: trials must be a scalar or one per observation")
            if not integer(n) or np.any(n < 0):
                raise ValueError("binomial_logit: trials must be integers >= 0")
            if not integer(y) or np.any(y < 0) or np.any(y > n):
                raise ValueError("binomial_logit: y must be integers with 0 <= y <= trials")
        elif L.trials is not None:
            raise ValueError(f"{L.dist}: trials belong to binomial_logit")
        if L.dist in DISPERSION_LIKS:
            if L.alpha is None:
                raise ValueError(f"{L.dist} needs alpha")
            if isinstance(L.alpha, Ref) and self.var(L.alpha.var).size != 1:
                raise ValueError(f"{L.dist}: alpha must be a scalar variable")
            self._check_scale(L.alpha, f"{L.dist}: alpha")
            if L.dist == "negative_binomial_log" and (not integer(y) or np.any(y < 0)):
                raise ValueError("negative_binomial_log: y must be integers >= 0")
            if L.dist == "gamma_log" and not (np.all(np.isfinite(y)) and np.all(y > 0)):
                raise ValueError("gamma_log: y must be > 0")
        elif L.alpha is not None:
            raise ValueError(f"{L.dist}: alpha belongs to the negative_binomial_log / gamma_log likelihoods")
        if L.dist in ("binomial_logit",) + DISPERSION_LIKS and L.sigma is not None:
            raise ValueError(f"{L.dist} has no sigma (its parameter is {'trials' if L.dist == 'binomial_logit' else 'alpha'})")

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
            out[v.rv_name] = x[..., 0] if v.size == 1 else x
        return out

    def eval_deterministics(self, posterior: dict) -> dict:
        """Deterministics from CONSTRAINED draws (``posterior``: rv name -> [..., size] or [...] for scalars, as ``constrain``
        returns them): value_i = sum_t coef_t[i] * prod_f x_f[idx_f[i]]."""
        out = {}
        for d in self.deterministics:
            lead = None
            total = 0.0
            for t in d.terms:
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
                if t.coef is not None and np.ndim(t.coef) in (1, 2):  # 2: a design term's X
                    out[f"{L.name}_coef{k}"] = np.asarray(t.coef)
                for vn, idx in t.factors:
                    if idx is not None:
                        out[f"{L.name}_{vn}_idx"] = np.asarray(idx)
            if L.trials is not None and np.ndim(L.trials) == 1:
                out[f"{L.name}_trials"] = np.asarray(L.trials)
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
        pars = [_param(ir, a, off) for a in p.params] + [(0, 0.0, -1)] * (3 - len(p.params))
        priors.append((PRIOR_DISTS[p.dist][0], index[ir.var(p.var).name], pars))
    liks = []
    for L in ir.likelihoods:
        # the likelihood's one parameter slot: sigma, or the trials / alpha of the count and positive families
        par = L.trials if L.dist == "binomial_logit" else (L.alpha if L.dist in DISPERSION_LIKS else L.sigma)
        liks.append(dict(dist=LIK_DISTS[L.dist], N=len(L.y), y=np.ascontiguousarray(L.y, dtype=np.float64),
                         terms=_lower_terms(ir, L.terms, len(L.y), off), nu=float(L.nu), y_var=0,
                         **_lower_slot(ir, par, off)))
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
    not changed."""
    out = copy.deepcopy(model)
    for L in out.likelihoods:
        L.terms = _fuse_terms(out, L.terms, len(L.y))
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

    pri = {ir.var(p.var).name: p for p in ir.priors}
    if len(pri) != len(ir.priors) or len(ir.likelihoods) != 1:
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
