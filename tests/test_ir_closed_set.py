"""Every factor of the model IR's closed set, on the device, against an independent high-precision reference.

``CASES`` is a catalogue of small models.  Together they hold every prior with every parameter kind the IR allows
(a constant, or a ``Ref`` to a location scalar, a log-scale or an interval scale) on every transform that keeps the
variable inside the prior's support; every likelihood with every kind of its parameter slot; the linear-predictor shapes
(a term with no factor, a scalar coefficient, one to three factors, broadcast / elementwise / indexed factors, an index
with an empty group or one dominant group, a variable in two terms and in two likelihoods); two likelihoods of different
lengths in one model; and AR(1) with constant or random phi and sigma, as a random walk, twice in one model.

``_mp_logp`` writes the joint log-density with mpmath at 40 digits from the published definitions (transform,
log-Jacobian, the sum of every factor with all its constants); the gradient is ``mpmath.diff`` per coordinate.  It reads
the ``ModelIR`` dataclasses and nothing else of the package or of oracle/.  Besides the value it returns
S = sum |additive pieces| (every elementwise term, split where a definition adds several parts), the scale a
correctly rounded double evaluation can be expected to reach: logp is compared to 1e-13 S, the gradient to
1e-12 max(1, |g|_inf).

Interval variables far out (|q| >= 12) are compared with the NumPy oracle only: there sigmoid(q) rounds next to 1 in the
device, the oracle and PyTensor alike, so dx/dq carries the same relative error 1e-12 .. 1e-8 in all three, and from
|q| ~ 30 on the variable rounds onto its bound.

CPU: the reference against scipy.stats, the oracle against the reference on every case, the support rule of
``ModelIR.validate()``.  GPU: the generic device function (chain = warp and, forced, chain = CTA) against both; every
(W, NPL) instantiation at the edges of its bucket; fixed-step NUTS against the oracle sampler; the pointwise
log-likelihood against scipy.stats; the same support rule in ``b200_model_create``."""
import re
import zlib
from functools import lru_cache

import mpmath
import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import stats
from scipy.special import expit
from test_frontend_mock import fake_pytensor  # noqa: F401

from pymc_b200 import ir
from pymc_b200.ir import AR1, Likelihood, ModelIR, Prior, Ref, Term, Var

MP_DPS = 40
LP_TOL, GRAD_TOL = 1e-13, 1e-12
SCALE_RULE = "must be a finite constant > 0 or a scalar variable with positive support"


# ------------------------------------------------------------------------------------------------------------------------
# the high-precision reference
# ------------------------------------------------------------------------------------------------------------------------
def _mp_prior_pieces(dist, x, a):
    """Additive pieces of log p(x) of one element under a prior with parameters a (mpf), every constant included."""
    pi = mp.pi
    if dist == "flat":
        return [mpf(0)]
    if dist == "normal":
        z = (x - a[0]) / a[1]
        return [-z * z / 2, -mp.log(a[1]), -mp.log(2 * pi) / 2]
    if dist == "halfnormal":
        z = x / a[0]
        return [-z * z / 2, -mp.log(a[0]), mp.log(2 / pi) / 2]
    if dist == "cauchy":
        return [-mp.log(pi), -mp.log(a[1]), -mp.log(1 + ((x - a[0]) / a[1]) ** 2)]
    if dist == "halfcauchy":
        return [mp.log(2 / pi), -mp.log(a[0]), -mp.log(1 + (x / a[0]) ** 2)]
    if dist == "exponential":
        return [mp.log(a[0]), -a[0] * x]
    if dist == "studentt":
        nu, z = a[0], (x - a[1]) / a[2]
        return [mp.loggamma((nu + 1) / 2), -mp.loggamma(nu / 2), -mp.log(nu * pi) / 2, -mp.log(a[2]),
                -(nu + 1) / 2 * mp.log(1 + z * z / nu)]
    if dist == "uniform":
        return [-mp.log(a[1] - a[0])]
    if dist == "gamma":
        return [a[0] * mp.log(a[1]), -mp.loggamma(a[0]), (a[0] - 1) * mp.log(x), -a[1] * x]
    if dist == "beta":
        return [(a[0] - 1) * mp.log(x), (a[1] - 1) * mp.log(1 - x), -mp.loggamma(a[0]), -mp.loggamma(a[1]),
                mp.loggamma(a[0] + a[1])]
    if dist == "lognormal":
        lx = mp.log(x)
        z = (lx - a[0]) / a[1]
        return [-z * z / 2, -lx, -mp.log(a[1]), -mp.log(2 * pi) / 2]
    raise NotImplementedError(dist)


def _mp_lik_pieces(dist, y, eta, s, nu):
    """Pieces of log p(y | eta) of one observation; s is sigma, the trials or the dispersion alpha."""
    if dist == "normal":
        return _mp_prior_pieces("normal", y, [eta, s])
    if dist == "studentt":
        return _mp_prior_pieces("studentt", y, [nu, eta, s])
    if dist == "normal_logvar":
        return _mp_prior_pieces("normal", y, [mpf(0), mp.exp(eta / 2)])
    lp, lq = -mp.log(1 + mp.exp(-eta)), -mp.log(1 + mp.exp(eta))  # log p, log(1 - p) of p = 1 / (1 + exp(-eta))
    if dist == "bernoulli_logit":
        return [y * lp, (1 - y) * lq]
    if dist == "binomial_logit":
        return [mp.loggamma(s + 1), -mp.loggamma(y + 1), -mp.loggamma(s - y + 1), y * lp, (s - y) * lq]
    mu = mp.exp(eta)
    if dist == "poisson_log" or (dist == "negative_binomial_log" and s > ir.NEGBIN_POISSON_ALPHA):
        return [y * eta, -mu, -mp.loggamma(y + 1)]
    if dist == "negative_binomial_log":  # n = alpha, p = alpha / (mu + alpha)
        return [mp.loggamma(y + s), -mp.loggamma(s), -mp.loggamma(y + 1), s * mp.log(s / (mu + s)), y * mp.log(mu / (mu + s))]
    if dist == "gamma_log":  # shape alpha, rate beta = alpha exp(-eta)
        b = s / mu
        return [s * mp.log(b), -mp.loggamma(s), (s - 1) * mp.log(y), -b * y]
    raise NotImplementedError(dist)


def _mp_constrain(m, q):
    """name -> constrained values, and the log-Jacobian pieces of every coordinate of q."""
    x, jac, o = {}, [], 0
    for v in m.vars:
        qv = q[o : o + v.size]
        o += v.size
        if v.transform == "log":
            x[v.name] = [mp.exp(t) for t in qv]
            jac += [[t] for t in qv]
        elif v.transform == "interval":
            lo, hi = mpf(v.bounds[0]), mpf(v.bounds[1])
            sg = [1 / (1 + mp.exp(-t)) for t in qv]
            x[v.name] = [lo + (hi - lo) * s for s in sg]
            jac += [[mp.log(hi - lo), mp.log(s), mp.log(s) - t] for s, t in zip(sg, qv)]  # 1 - sg = sg exp(-q)
        else:
            x[v.name] = list(qv)
            jac += [[] for _ in qv]
    return x, jac


def _mp_factors(m):
    """[(names of the variables a factor reads, x -> its additive pieces)]"""
    name = lambda r: m.var(r).name  # noqa: E731
    par = lambda a, x: x[name(a.var)][0] if isinstance(a, Ref) else mpf(float(a))  # noqa: E731
    refs = lambda *ps: {name(a.var) for a in ps if isinstance(a, Ref)}  # noqa: E731
    out = []
    for p in m.priors:
        vn = name(p.var)
        out.append(({vn} | refs(*p.params),
                    lambda x, p=p, vn=vn: [t for xi in x[vn] for t in _mp_prior_pieces(p.dist, xi, [par(a, x) for a in p.params])]))
    for L in m.likelihoods:
        N = len(L.y)
        y = [mpf(float(v)) for v in L.y]
        terms = [([mpf(1)] * N if t.coef is None else [mpf(float(c)) for c in np.broadcast_to(t.coef, (N,))],
                  [(name(vn), idx) for vn, idx in t.factors]) for t in L.terms]
        slot = L.trials if L.dist == "binomial_logit" else (L.alpha if L.alpha is not None else L.sigma)
        obs = [mpf(float(v)) for v in slot] if slot is not None and not isinstance(slot, Ref) and np.ndim(slot) == 1 else None

        def lik(x, L=L, y=y, terms=terms, slot=slot, obs=obs, N=N):
            eta = [mpf(0)] * N
            for coef, fs in terms:
                for i in range(N):
                    pr = coef[i]
                    for vn, idx in fs:
                        xv = x[vn]
                        pr *= xv[int(idx[i])] if idx is not None else (xv[0] if len(xv) == 1 else xv[i])
                    eta[i] += pr
            s = [mpf(1)] * N if slot is None else ([par(slot, x)] * N if isinstance(slot, Ref) or np.ndim(slot) == 0 else obs)
            return [t for i in range(N) for t in _mp_lik_pieces(L.dist, y[i], eta[i], s[i], mpf(float(L.nu)))]
        out.append(({vn for _, fs in terms for vn, _ in fs} | refs(L.sigma, L.alpha), lik))
    for a in m.ar1:
        vn = name(a.var)

        def ar(x, a=a, vn=vn):
            h, phi, sg = x[vn], par(a.phi, x), par(a.sigma, x)
            return _mp_prior_pieces("normal", h[0], [mpf(0), mpf(float(a.init_sigma))]) + \
                [t for k in range(1, len(h)) for t in _mp_prior_pieces("normal", h[k], [phi * h[k - 1], sg])]
        out.append(({vn} | refs(a.phi, a.sigma), ar))
    return out


def _mp_logp(m, q):
    """(logp, S = sum of |additive pieces|) at the unconstrained point q, with 40 significant digits."""
    with mp.workdps(MP_DPS):
        x, jac = _mp_constrain(m, [mpf(float(t)) for t in q])
        pieces = [t for j in jac for t in j] + [t for _, f in _mp_factors(m) for t in f(x)]
        return float(mp.fsum(pieces)), float(mp.fsum(abs(t) for t in pieces))


def _mp_grad(m, q):
    """d logp / dq by mpmath.diff per coordinate, through the factors that read the coordinate's variable."""
    facs, off, g = _mp_factors(m), m.offsets(), np.empty(m.n)
    with mp.workdps(MP_DPS):
        q0 = [mpf(float(t)) for t in q]
        for v in m.vars:
            fs = [f for deps, f in facs if v.name in deps]
            for j in range(off[v.name], off[v.name] + v.size):
                def h(t, j=j, fs=fs):
                    qq = q0[:]
                    qq[j] = t
                    x, jac = _mp_constrain(m, qq)
                    return mp.fsum(jac[j] + [p for f in fs for p in f(x)])
                g[j] = float(mpmath.diff(h, q0[j]))
    return g


# ------------------------------------------------------------------------------------------------------------------------
# the case catalogue
# ------------------------------------------------------------------------------------------------------------------------
def _ref_var(kind):
    """The scalar a Ref parameter points at: a location, a log-scale or an interval scale, with its own prior."""
    return {"loc": (Var("m", "m", 1), Prior("normal", "m", (0.5, 1.0))),
            "log": (Var("s_log__", "s", 1, "log"), Prior("halfnormal", "s_log__", (1.5,))),
            "int": (Var("w_interval__", "w", 1, "interval", (0.1, 4.0)), Prior("uniform", "w_interval__", (0.1, 4.0)))}[kind]


def _with_refs(kinds, vars_, priors):
    for k in dict.fromkeys(kinds):
        v, p = _ref_var(k)
        vars_.append(v)
        priors.append(p)


def _ref(kind):
    return Ref(_ref_var(kind)[0].name)


PRIOR_SPECS = [  # (dist, transform, bounds, parameters: a constant, or the kind of scalar a Ref points at)
    ("normal", None, None, (0.3, 1.7)), ("normal", None, None, ("loc", "log")), ("normal", None, None, (-0.4, "int")),
    ("cauchy", None, None, (-0.2, 2.0)), ("cauchy", None, None, ("loc", "log")), ("cauchy", None, None, (0.1, "int")),
    ("studentt", None, None, (4.0, 0.5, 1.2)), ("studentt", None, None, (3.0, "loc", "log")),
    ("studentt", None, None, (7.0, 0.0, "int")),
    ("flat", None, None, ()), ("flat", "log", None, ()),
    ("halfnormal", "log", None, (1.3,)), ("halfnormal", "log", None, ("log",)), ("halfnormal", "interval", (0.0, 4.0), ("int",)),
    ("halfcauchy", "log", None, (2.5,)), ("halfcauchy", "interval", (0.0, 6.0), ("log",)), ("halfcauchy", "log", None, ("int",)),
    ("exponential", "log", None, (3.0,)), ("exponential", "interval", (0.0, 3.0), ("log",)),
    ("exponential", "log", None, ("int",)),
    ("gamma", "log", None, (2.5, 1.5)), ("gamma", "interval", (0.0, 10.0), (0.8, 2.0)),
    ("lognormal", "log", None, (0.2, 0.7)), ("lognormal", "log", None, ("loc", "log")),
    ("lognormal", "interval", (0.0, 20.0), (0.5, "int")),
    ("beta", "interval", (0.0, 1.0), (2.0, 3.5)), ("beta", "interval", (0.2, 0.9), (0.7, 1.5)),
    ("uniform", "interval", (-1.0, 3.0), (-1.0, 3.0)), ("uniform", "interval", (0.0, 2.0), (-1.0, 3.0)),
]


def _prior_id(dist, tr, bounds, params):
    t = "none" if tr is None else (tr if bounds is None else f"interval{bounds[0]:g}_{bounds[1]:g}")
    return f"prior-{dist}-{t}-" + ("_".join(p if isinstance(p, str) else "c" for p in params) or "noparams")


def _prior_case(dist, tr, bounds, params, rng):
    """The prior on a 3-vector x (which a Normal likelihood observes elementwise), its Ref parameters' scalars."""
    vars_, priors = [Var("x", "x", 3, tr, bounds)], []
    _with_refs([p for p in params if isinstance(p, str)], vars_, priors)
    priors.insert(0, Prior(dist, "x", tuple(_ref(p) if isinstance(p, str) else p for p in params)))
    y = rng.normal(1.0, 0.5, 3)
    return ModelIR(vars=vars_, priors=priors, likelihoods=[Likelihood("normal", y, [Term([("x", None)])], sigma=1.3)])


def _regression(rng, N, slot_kinds=()):
    """b0 + b1 x_i over N observations: the variables, priors and terms, plus the Ref scalars named by slot_kinds."""
    x = rng.standard_normal(N)
    vars_ = [Var("b0", "b0", 1), Var("b1", "b1", 1)]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "b1", (0.0, 1.0))]
    _with_refs(slot_kinds, vars_, priors)
    return x, vars_, priors, [Term([("b0", None)]), Term([("b1", None)], coef=x)]


def _y(dist, eta, rng, slot=None):
    if dist in ("normal", "studentt"):
        return eta + 0.8 * rng.standard_normal(len(eta))
    if dist == "normal_logvar":
        return np.exp(eta / 2) * rng.standard_normal(len(eta))
    if dist == "bernoulli_logit":
        return (rng.random(len(eta)) < expit(eta)).astype(float)
    if dist == "poisson_log":
        return rng.poisson(np.exp(eta)).astype(float)
    if dist == "binomial_logit":
        return rng.binomial(np.broadcast_to(slot, eta.shape).astype(int), expit(eta)).astype(float)
    if dist == "negative_binomial_log":
        return rng.negative_binomial(2.0, 2.0 / (np.exp(eta) + 2.0)).astype(float)
    return rng.gamma(2.0, np.exp(eta) / 2.0)


def _lik_case(dist, kind, rng, N=40, nu=0.0, shape="plain"):
    """One likelihood with the parameter slot `kind` (const / ref_log / ref_int / obs / none) under a term shape."""
    refs = {"ref_log": ["log"], "ref_int": ["int"]}.get(kind, [])
    N = 24 if shape == "elementwise" else N
    x, vars_, priors, terms = _regression(rng, N, refs)
    eta0 = 0.5 + 0.4 * x
    if shape == "three_factors":  # + 0.5 s a[g] b1: a product of a log-scale, an indexed vector and a scalar
        g = rng.integers(0, 5, N).astype(np.int32)
        vars_ += [Var("a", "a", 5), Var("sa_log__", "sa", 1, "log")]
        priors += [Prior("normal", "a", (0.0, 1.0)), Prior("halfcauchy", "sa_log__", (1.0,))]
        terms.append(Term([("sa_log__", None), ("a", g), ("b1", None)], coef=0.5))
    elif shape in ("empty_group", "dominant_group"):
        G = 7
        if shape == "empty_group":  # groups 2 and 6 have no observations
            g = rng.choice([0, 1, 3, 4, 5], N).astype(np.int32)
        else:  # 90 % of the observations in group 3
            g = np.where(rng.random(N) < 0.9, 3, rng.integers(0, G, N)).astype(np.int32)
        vars_.append(Var("a", "a", G))
        priors.append(Prior("normal", "a", (0.0, 0.5)))
        terms.append(Term([("a", g)]))
    elif shape == "elementwise":  # a vector of the likelihood's own length, no index
        vars_.append(Var("e", "e", N))
        priors.append(Prior("normal", "e", (0.0, 0.3)))
        terms.append(Term([("e", None)]))
    elif shape == "offset_and_scalar_coef":  # a term with no factor (a constant offset) and a scalar coefficient
        terms = [Term([], coef=0.2 * rng.standard_normal(N)), Term([("b0", None)], coef=0.7), terms[1]]
    slot = {"const": 1.4, "ref_log": _ref("log"), "ref_int": _ref("int"), "obs": np.exp(rng.uniform(-0.5, 0.5, N)),
            "none": None}[kind]
    kw = {}
    if dist in ("normal", "studentt"):
        kw = dict(sigma=slot, nu=nu)
    elif dist == "binomial_logit":
        slot = 12.0 if kind == "const" else rng.integers(0, 25, N).astype(float)
        kw = dict(trials=slot)
    elif dist in ir.DISPERSION_LIKS:
        kw = dict(alpha=2.5 if kind == "const" else slot)
    y = _y(dist, eta0, rng, slot)
    return ModelIR(vars=vars_, priors=priors, likelihoods=[Likelihood(dist, y, terms, **kw)])


def _studentt_outlier(rng):
    m = _lik_case("studentt", "const", rng, nu=4.0)
    m.likelihoods[0].y[0] += 1e6 * 1.4  # a residual of 1e6 sigma
    return m


def _shared_variable(rng):
    """b1 in two terms of one likelihood and in a second likelihood."""
    N1, N2 = 36, 14
    x1, x2 = rng.standard_normal(N1), rng.standard_normal(N2)
    vars_ = [Var("b0", "b0", 1), Var("b1", "b1", 1), Var("s_log__", "s", 1, "log")]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "b1", (0.0, 1.0)), Prior("exponential", "s_log__", (1.0,))]
    t1 = [Term([("b0", None)]), Term([("b1", None)], coef=x1), Term([("b1", None), ("s_log__", None)], coef=0.3 * x1 ** 2)]
    t2 = [Term([("b1", None)], coef=x2)]
    return ModelIR(vars=vars_, priors=priors, likelihoods=[
        Likelihood("normal", 0.5 + 0.4 * x1 + rng.standard_normal(N1), t1, sigma=Ref("s_log__"), name="y1"),
        Likelihood("poisson_log", rng.poisson(np.exp(0.3 * x2)).astype(float), t2, name="y2")])


def _two_likelihoods(rng):
    """A Normal likelihood of 50 observations and a Bernoulli one of 20 sharing a group effect: the second reuses the
    team's residual scratch the first has filled further."""
    N1, N2, G = 50, 20, 6
    g1, g2 = rng.integers(0, G, N1).astype(np.int32), rng.integers(0, G, N2).astype(np.int32)
    x1 = rng.standard_normal(N1)
    vars_ = [Var("mu", "mu", 1), Var("tau_log__", "tau", 1, "log"), Var("z", "z", G), Var("b", "b", 1),
             Var("eps_log__", "eps", 1, "log")]
    priors = [Prior("normal", "mu", (0.0, 2.0)), Prior("halfnormal", "tau_log__", (1.0,)), Prior("normal", "z", (0.0, 1.0)),
              Prior("normal", "b", (0.0, 1.0)), Prior("halfcauchy", "eps_log__", (1.0,))]
    a = rng.normal(0.0, 0.7, G)
    return ModelIR(vars=vars_, priors=priors, likelihoods=[
        Likelihood("normal", a[g1] + 0.5 * x1 + 0.6 * rng.standard_normal(N1),
                   [Term([("mu", None)]), Term([("tau_log__", None), ("z", g1)]), Term([("b", None)], coef=x1)],
                   sigma=Ref("eps_log__"), name="y1"),
        Likelihood("bernoulli_logit", (rng.random(N2) < expit(a[g2])).astype(float),
                   [Term([("mu", None)]), Term([("tau_log__", None), ("z", g2)])], name="y2")])


def _ar1_case(kind, rng):
    T = 14 if kind == "two" else 20
    vars_ = [Var("h", "h", T)]
    priors = []
    if kind == "const":
        a = [AR1("h", 0.6, 0.8, 1.0)]
    elif kind == "random_walk":  # phi = 1: a Gaussian random walk, sigma a Ref to an interval scale
        _with_refs(["int"], vars_, priors)
        a = [AR1("h", 1.0, _ref("int"), 0.5)]
    elif kind == "ref":
        vars_ += [Var("phi_interval__", "phi", 1, "interval", (-1.0, 1.0)), Var("sigma_log__", "sigma", 1, "log", initial=np.log(0.3))]
        priors += [Prior("uniform", "phi_interval__", (-1.0, 1.0)), Prior("exponential", "sigma_log__", (2.0,))]
        a = [AR1("h", Ref("phi_interval__"), Ref("sigma_log__"), 1.0)]
    else:  # two AR(1) factors: one with a random phi and constant sigma, one with constant phi and a random sigma
        vars_ += [Var("k", "k", T - 5), Var("phi_interval__", "phi", 1, "interval", (-1.0, 1.0)), Var("s_log__", "s", 1, "log")]
        priors += [Prior("uniform", "phi_interval__", (-1.0, 1.0)), Prior("halfnormal", "s_log__", (1.0,))]
        a = [AR1("h", Ref("phi_interval__"), 0.7, 1.0), AR1("k", -0.3, Ref("s_log__"), 2.0)]
    h = np.cumsum(rng.normal(0.0, 0.3, T))
    if kind == "ref":  # the stochastic-volatility observation on mu + h
        vars_.insert(0, Var("mu", "mu", 1))
        priors.insert(0, Prior("normal", "mu", (0.0, 5.0)))
        liks = [Likelihood("normal_logvar", np.exp(h / 2) * rng.standard_normal(T), [Term([("mu", None)]), Term([("h", None)])])]
    else:
        liks = [Likelihood("normal", h + 0.5 * rng.standard_normal(T), [Term([("h", None)])], sigma=0.5)]
        if kind == "two":
            liks.append(Likelihood("normal", rng.standard_normal(T - 5), [Term([("k", None)])], sigma=0.9, name="yk"))
    return ModelIR(vars=vars_, priors=priors, likelihoods=liks, ar1=a)


LIK_SPECS = [  # (case id, dist, slot kind, nu, term shape)
    ("lik-normal-const", "normal", "const", 0.0, "plain"),
    ("lik-normal-ref_log", "normal", "ref_log", 0.0, "plain"),
    ("lik-normal-ref_int", "normal", "ref_int", 0.0, "plain"),
    ("lik-normal-obs", "normal", "obs", 0.0, "plain"),
    ("lik-studentt-nu1-const", "studentt", "const", 1.0, "plain"),
    ("lik-studentt-nu4-ref_log", "studentt", "ref_log", 4.0, "plain"),
    ("lik-studentt-nu30-obs", "studentt", "obs", 30.0, "plain"),
    ("lik-studentt-nu4-ref_int", "studentt", "ref_int", 4.0, "plain"),
    ("lik-bernoulli", "bernoulli_logit", "none", 0.0, "plain"),
    ("lik-poisson", "poisson_log", "none", 0.0, "plain"),
    ("lik-normal_logvar", "normal_logvar", "none", 0.0, "plain"),
    ("lik-binomial-obs-three_factors", "binomial_logit", "obs", 0.0, "three_factors"),
    ("lik-binomial-const-empty_group", "binomial_logit", "const", 0.0, "empty_group"),
    ("lik-negbin-const-empty_group", "negative_binomial_log", "const", 0.0, "empty_group"),
    ("lik-negbin-ref_log-dominant_group", "negative_binomial_log", "ref_log", 0.0, "dominant_group"),
    ("lik-negbin-ref_int-three_factors", "negative_binomial_log", "ref_int", 0.0, "three_factors"),
    ("lik-gamma-const-elementwise", "gamma_log", "const", 0.0, "elementwise"),
    ("lik-gamma-ref_log-offset_and_scalar_coef", "gamma_log", "ref_log", 0.0, "offset_and_scalar_coef"),
    ("lik-gamma-ref_int-dominant_group", "gamma_log", "ref_int", 0.0, "dominant_group"),
    ("terms-normal-offset_and_scalar_coef", "normal", "ref_log", 0.0, "offset_and_scalar_coef"),
    ("terms-poisson-three_factors", "poisson_log", "none", 0.0, "three_factors"),
    ("terms-studentt-elementwise", "studentt", "const", 4.0, "elementwise"),
    ("terms-bernoulli-dominant_group", "bernoulli_logit", "none", 0.0, "dominant_group"),
]

CASES = {_prior_id(*s): (lambda rng, s=s: _prior_case(*s, rng)) for s in PRIOR_SPECS}
CASES.update({cid: (lambda rng, s=s: _lik_case(s[0], s[1], rng, nu=s[2], shape=s[3])) for cid, *s in LIK_SPECS})
CASES.update({
    "lik-studentt-nu4-outlier": _studentt_outlier,
    "terms-shared_variable-two_likelihoods": _shared_variable,
    "two_likelihoods-normal50-bernoulli20": _two_likelihoods,
    "ar1-const": lambda rng: _ar1_case("const", rng),
    "ar1-ref-stochvol": lambda rng: _ar1_case("ref", rng),
    "ar1-random_walk": lambda rng: _ar1_case("random_walk", rng),
    "ar1-two": lambda rng: _ar1_case("two", rng),
})
# points beyond the generic ones, as {variable: unconstrained value}: a predictor at the edges of the link functions
CASE_EDGES = {"lik-bernoulli": [{"b0": 40.0}, {"b0": -40.0}], "lik-poisson": [{"b0": 20.0}, {"b0": -20.0}]}


def build(cid):
    return CASES[cid](np.random.default_rng(zlib.crc32(cid.encode())))


def _set(m, q, values):
    q, off = q.copy(), m.offsets()
    for vn, val in values.items():
        v = m.var(vn)
        q[off[v.name] : off[v.name] + v.size] = val
    return q


def points(m, cid):
    """The case's initial point + U(-1.5, 1.5) (twice), log-scales at -12 / +12, intervals at -8 / +8, its own edges."""
    rng = np.random.default_rng(zlib.crc32(cid.encode()) + 1)
    q0 = m.initial_point()
    Q = [q0 + rng.uniform(-1.5, 1.5, m.n) for _ in range(2)]
    for tr, e in (("log", 12.0), ("interval", 8.0)):
        names = {v.name: None for v in m.vars if v.transform == tr}
        Q += [_set(m, q0, dict.fromkeys(names, s * e)) for s in (-1, 1) if names]
    Q += [_set(m, q0, edge) for edge in CASE_EDGES.get(cid, [])]
    return np.array(Q)


def far_interval_points(m):
    names = [v.name for v in m.vars if v.transform == "interval"]
    q0 = m.initial_point()
    return np.array([_set(m, q0, dict.fromkeys(names, s * e)) for e in (12.0, 20.0, 30.0) for s in (-1, 1)]) if names else None


@lru_cache(maxsize=None)
def mp_reference(cid):
    """(Q, logp, S, grad) of the mp reference at the case's points; computed once per session."""
    m = build(cid)
    Q = points(m, cid)
    lp, S = np.array([_mp_logp(m, q) for q in Q]).T
    return Q, lp, S, np.array([_mp_grad(m, q) for q in Q])


def assert_close_to_reference(lp, g, ref_lp, S, ref_g, what):
    assert np.all(np.abs(lp - ref_lp) <= LP_TOL * S), (what, np.abs(lp - ref_lp) / S)
    scale = np.maximum(1.0, np.max(np.abs(ref_g), axis=1))
    err = np.max(np.abs(g - ref_g), axis=1) / scale
    assert np.all(err <= GRAD_TOL), (what, err)


CASE_IDS = list(CASES)


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference, the catalogue and the oracle
# ------------------------------------------------------------------------------------------------------------------------
def _scipy_prior(dist, p):
    return {"normal": lambda x: stats.norm(p[0], p[1]).logpdf(x), "halfnormal": lambda x: stats.halfnorm(scale=p[0]).logpdf(x),
            "cauchy": lambda x: stats.cauchy(p[0], p[1]).logpdf(x), "halfcauchy": lambda x: stats.halfcauchy(scale=p[0]).logpdf(x),
            "exponential": lambda x: stats.expon(scale=1 / p[0]).logpdf(x), "studentt": lambda x: stats.t(p[0], p[1], p[2]).logpdf(x),
            "uniform": lambda x: stats.uniform(p[0], p[1] - p[0]).logpdf(x), "gamma": lambda x: stats.gamma(p[0], scale=1 / p[1]).logpdf(x),
            "beta": lambda x: stats.beta(p[0], p[1]).logpdf(x),
            "lognormal": lambda x: stats.lognorm(p[1], scale=np.exp(p[0])).logpdf(x)}[dist]


def scipy_loglik(dist, y, eta, s, nu):
    """log p(y_i | eta_i) from scipy.stats; s is sigma, the trials or alpha."""
    if dist == "normal":
        return stats.norm.logpdf(y, eta, s)
    if dist == "studentt":
        return stats.t.logpdf(y, nu, eta, s)
    if dist == "normal_logvar":
        return stats.norm.logpdf(y, 0.0, np.exp(eta / 2))
    if dist == "bernoulli_logit":
        return stats.bernoulli.logpmf(y, expit(eta))
    if dist == "poisson_log":
        return stats.poisson.logpmf(y, np.exp(eta))
    if dist == "binomial_logit":
        return stats.binom.logpmf(y, s, expit(eta))
    if dist == "negative_binomial_log":
        return stats.nbinom.logpmf(y, s, s / (np.exp(eta) + s))
    return stats.gamma.logpdf(y, s, scale=np.exp(eta) / s)


PRIOR_PINS = [("normal", (0.3, 1.7), [-4.0, 0.1, 9.0]), ("halfnormal", (1.3,), [1e-6, 0.7, 12.0]),
              ("cauchy", (-0.2, 2.0), [-300.0, 0.5, 1e4]), ("halfcauchy", (2.5,), [1e-5, 3.0, 1e5]),
              ("exponential", (3.0,), [1e-6, 0.4, 40.0]), ("studentt", (4.0, 0.5, 1.2), [-1e6, 0.3, 25.0]),
              ("studentt", (1.0, 0.0, 1.0), [-3.0, 1e3]), ("studentt", (30.0, -1.0, 0.5), [0.0, 7.0]),
              ("uniform", (-1.0, 3.0), [-0.5, 2.9]), ("gamma", (2.5, 1.5), [1e-4, 1.0, 30.0]), ("gamma", (0.8, 2.0), [1e-3, 5.0]),
              ("beta", (2.0, 3.5), [1e-4, 0.5, 0.9997]), ("beta", (0.7, 1.5), [0.01, 0.6]),
              ("lognormal", (0.2, 0.7), [1e-3, 1.0, 1.6e5])]


@pytest.mark.parametrize("dist,params,xs", PRIOR_PINS, ids=[f"{d}-{k}" for k, (d, *_) in enumerate(PRIOR_PINS)])
def test_mp_prior_terms_equal_scipy(dist, params, xs):
    for x in xs:
        want = float(_scipy_prior(dist, params)(x))
        with mp.workdps(MP_DPS):
            got = float(mp.fsum(_mp_prior_pieces(dist, mpf(x), [mpf(p) for p in params])))
        assert abs(got - want) <= 1e-13 * max(1.0, abs(want)), (dist, x, got, want)


LIK_PINS = [("normal", [(0.3, -0.2, 0.9), (50.0, 1.0, 0.01)]), ("studentt", [(0.3, -0.2, 0.9), (1.4e6, 0.0, 1.4)]),
            ("normal_logvar", [(0.4, -1.0, None), (-2.0, 3.0, None)]), ("bernoulli_logit", [(1.0, 2.5, None), (0.0, -4.0, None)]),
            ("poisson_log", [(3.0, 1.1, None), (0.0, -2.0, None), (7.0, 20.0, None)]),
            ("binomial_logit", [(3.0, 0.4, 12.0), (0.0, -1.0, 7.0), (20.0, 2.0, 20.0)]),
            ("negative_binomial_log", [(0.0, 0.3, 2.5), (17.0, 2.0, 0.4), (4.0, 1.0, 40.0)]),
            ("gamma_log", [(0.7, 0.2, 2.5), (12.0, 1.5, 0.3), (2.0, 0.5, 1.6e5)])]


@pytest.mark.parametrize("dist,rows", LIK_PINS, ids=[d for d, _ in LIK_PINS])
def test_mp_likelihood_terms_equal_scipy(dist, rows):
    for nu in ((1.0, 4.0, 30.0) if dist == "studentt" else (0.0,)):
        for y, eta, s in rows:
            s = 1.0 if s is None else s
            want = float(scipy_loglik(dist, np.array([y]), np.array([eta]), s, nu)[0])
            with mp.workdps(MP_DPS):
                got = float(mp.fsum(_mp_lik_pieces(dist, mpf(y), mpf(eta), mpf(s), mpf(nu))))
            assert abs(got - want) <= 1e-13 * max(1.0, abs(want)), (dist, y, eta, s, nu, got, want)


def test_mp_reference_gradient_and_jacobians_by_independent_means():
    """The mp joint density on a model with every transform equals scipy.stats plus the log-Jacobians written out, and
    mpmath.diff agrees with a high-order mp central difference."""
    m = ModelIR(vars=[Var("a", "a", 2), Var("s_log__", "s", 1, "log"), Var("p_interval__", "p", 1, "interval", (0.2, 0.9))],
                priors=[Prior("normal", "a", (0.1, Ref("s_log__"))), Prior("halfnormal", "s_log__", (1.5,)),
                        Prior("beta", "p_interval__", (0.7, 1.5))],
                likelihoods=[Likelihood("normal", np.array([0.3, -0.4, 1.1]), [Term([("a", np.array([0, 1, 1]))])],
                                        sigma=Ref("p_interval__"))])
    q = np.array([0.4, -0.8, 0.3, 1.7])
    lp, S = _mp_logp(m, q)
    s, sg = np.exp(q[2]), expit(q[3])
    p = 0.2 + 0.7 * sg
    want = (stats.norm(0.1, s).logpdf(q[:2]).sum() + stats.halfnorm(scale=1.5).logpdf(s) + q[2]
            + stats.beta(0.7, 1.5).logpdf(p) + np.log(0.7 * sg * (1 - sg))
            + stats.norm(q[[0, 1, 1]], p).logpdf([0.3, -0.4, 1.1]).sum())
    assert abs(lp - want) <= 1e-13 * S and S > abs(lp)
    g, h = _mp_grad(m, q), 1e-3
    for j in range(m.n):  # fourth-order central differences of the (double-rounded) reference value
        f = lambda t: _mp_logp(m, np.where(np.arange(m.n) == j, t, q))[0]  # noqa: E731
        fd = (-f(q[j] + 2 * h) + 8 * f(q[j] + h) - 8 * f(q[j] - h) + f(q[j] - 2 * h)) / (12 * h)
        assert abs(fd - g[j]) <= 1e-8 * max(1.0, abs(g[j])), j


def test_the_catalogue_covers_the_closed_set():
    """Every prior on every support-keeping transform kind with every parameter kind, every likelihood with every slot
    kind, and the predictor / model shapes, each in some case; the cases stay small."""
    priors, liks, shapes = set(), set(), set()
    for cid in CASE_IDS:
        m = build(cid)
        m.validate()
        assert m.n <= 32 and all(len(L.y) <= 60 for L in m.likelihoods), cid
        for p in m.priors:
            v = m.var(p.var)
            priors.add((p.dist, v.transform, "ref" if any(isinstance(a, Ref) for a in p.params) else "const"))
            for a in p.params:
                if isinstance(a, Ref):
                    priors.add((p.dist, "param", m.var(a.var).transform))
        for L in m.likelihoods:
            par = L.trials if L.dist == "binomial_logit" else (L.alpha if L.alpha is not None else L.sigma)
            kind = "none" if par is None else ("ref_" + m.var(par.var).transform if isinstance(par, Ref) else
                                               ("obs" if np.ndim(par) == 1 else "const"))
            liks.add((L.dist, kind) + ((L.nu,) if L.dist == "studentt" else ()))
            for t in L.terms:
                shapes.add(("factors", len(t.factors)))
                shapes.add(("coef", "none" if t.coef is None else ("scalar" if np.ndim(t.coef) == 0 else "array")))
                for vn, idx in t.factors:
                    v = m.var(vn)
                    shapes.add(("factor", "indexed" if idx is not None else ("broadcast" if v.size == 1 else "elementwise")))
                    if idx is not None:
                        counts = np.bincount(idx, minlength=v.size)
                        shapes.add(("empty group", bool(np.any(counts == 0))))
                        shapes.add(("dominant group", bool(np.max(counts) >= 0.85 * len(idx))))
        if len(m.likelihoods) == 2 and len(m.likelihoods[0].y) > len(m.likelihoods[1].y):
            shapes.add(("two likelihoods", "N1 > N2"))
            used = [{m.var(vn).name for t in L.terms for vn, _ in t.factors} for L in m.likelihoods]
            shapes.add(("shared across likelihoods", bool(used[0] & used[1])))
        for L in m.likelihoods:
            names = [m.var(vn).name for t in L.terms for vn, _ in t.factors]
            shapes.add(("variable in two terms", len(names) > len(set(names))))
        shapes.add(("ar1 factors", len(m.ar1)))
        for a in m.ar1:
            shapes.add(("ar1 phi", "ref" if isinstance(a.phi, Ref) else ("one" if a.phi == 1.0 else "const")))
            shapes.add(("ar1 sigma", "ref" if isinstance(a.sigma, Ref) else "const"))
    for d in ("normal", "cauchy", "studentt", "flat"):
        assert (d, None, "const") in priors, d
    for d in ("halfnormal", "halfcauchy", "exponential", "gamma", "lognormal"):
        assert any(k[:2] == (d, "log") for k in priors) and any(k[:2] == (d, "interval") for k in priors), d
    assert ("beta", "interval", "const") in priors and ("uniform", "interval", "const") in priors
    for d in ("normal", "cauchy", "studentt", "lognormal"):
        assert {(d, "param", None), (d, "param", "log"), (d, "param", "interval")} <= priors, d
    for d in ("halfnormal", "halfcauchy", "exponential"):
        assert {(d, "param", "log"), (d, "param", "interval"), (d, "log", "const")} <= priors, d
    for d in ("normal", "studentt"):
        assert {k[1] for k in liks if k[0] == d} >= {"const", "ref_log", "ref_interval", "obs"}, d
    assert {k[2] for k in liks if k[0] == "studentt"} >= {1.0, 4.0, 30.0}
    assert {("bernoulli_logit", "none"), ("poisson_log", "none"), ("normal_logvar", "none"),
            ("binomial_logit", "const"), ("binomial_logit", "obs")} <= liks
    for d in ir.DISPERSION_LIKS:
        assert {k[1] for k in liks if k[0] == d} >= {"const", "ref_log", "ref_interval"}, d
    assert {("factors", 0), ("factors", 1), ("factors", 2), ("factors", 3), ("coef", "scalar"), ("coef", "array"),
            ("factor", "indexed"), ("factor", "broadcast"), ("factor", "elementwise"), ("empty group", True),
            ("dominant group", True), ("two likelihoods", "N1 > N2"), ("shared across likelihoods", True),
            ("variable in two terms", True), ("ar1 factors", 2), ("ar1 phi", "ref"), ("ar1 phi", "one"), ("ar1 phi", "const"),
            ("ar1 sigma", "ref"), ("ar1 sigma", "const")} <= shapes


@pytest.mark.parametrize("cid", CASE_IDS)
def test_oracle_matches_the_mp_reference(cid):
    from oracle import ir_numpy_families

    m = build(cid)
    Q, lp_mp, S, g_mp = mp_reference(cid)
    f = ir_numpy_families.make_logp(m)
    lp = np.array([f(q)[0] for q in Q])
    g = np.array([f(q)[1] for q in Q])
    assert_close_to_reference(lp, g, lp_mp, S, g_mp, cid)


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the support rule
# ------------------------------------------------------------------------------------------------------------------------
def _one_prior(dist, params, tr=None, bounds=None, extra=()):
    vars_ = [Var("x", "x", 2, tr, bounds), Var("m", "m", 1), Var("s_log__", "s", 1, "log")] + list(extra)
    return ModelIR(vars=vars_, priors=[Prior(dist, "x", params)])


def _one_lik(dist, y, **kw):
    vars_ = [Var("b", "b", 1), Var("m", "m", 1), Var("s_log__", "s", 1, "log"), Var("h", "h", 4)]
    return ModelIR(vars=vars_, likelihoods=[Likelihood(dist, np.asarray(y, dtype=float), [Term([("b", None)])], **kw)])


def _one_ar1(phi, sigma, init_sigma=1.0):
    return ModelIR(vars=[Var("h", "h", 5), Var("m", "m", 1), Var("s_log__", "s", 1, "log")], ar1=[AR1("h", phi, sigma, init_sigma)])


OUT_OF_SUPPORT = [  # (what, model, the message both validate() and b200_model_create give)
    ("halfnormal untransformed", lambda: _one_prior("halfnormal", (1.0,)), "needs a log transform or an interval with lo >= 0"),
    ("halfcauchy on an interval below 0", lambda: _one_prior("halfcauchy", (1.0,), "interval", (-1.0, 2.0)),
     "needs a log transform or an interval with lo >= 0"),
    ("exponential untransformed", lambda: _one_prior("exponential", (1.0,)), "needs a log transform or an interval with lo >= 0"),
    ("gamma untransformed", lambda: _one_prior("gamma", (2.0, 1.0)), "needs a log transform or an interval with lo >= 0"),
    ("lognormal untransformed", lambda: _one_prior("lognormal", (0.0, 1.0)), "needs a log transform or an interval with lo >= 0"),
    ("beta on a log transform", lambda: _one_prior("beta", (2.0, 2.0), "log"), "needs an interval inside [0, 1]"),
    ("beta on (0, 2)", lambda: _one_prior("beta", (2.0, 2.0), "interval", (0.0, 2.0)), "needs an interval inside [0, 1]"),
    ("uniform untransformed", lambda: _one_prior("uniform", (0.0, 1.0)), "needs an interval inside the Uniform bounds"),
    ("uniform on a wider interval", lambda: _one_prior("uniform", (0.0, 1.0), "interval", (-0.5, 1.0)),
     "needs an interval inside the Uniform bounds"),
    ("normal sigma on an untransformed scalar", lambda: _one_prior("normal", (0.0, Ref("m"))), SCALE_RULE),
    ("normal sigma -1", lambda: _one_prior("normal", (0.0, -1.0)), SCALE_RULE),
    ("halfnormal sigma 0", lambda: _one_prior("halfnormal", (0.0,), "log"), SCALE_RULE),
    ("cauchy beta infinite", lambda: _one_prior("cauchy", (0.0, np.inf)), SCALE_RULE),
    ("halfcauchy beta on an untransformed scalar", lambda: _one_prior("halfcauchy", (Ref("m"),), "log"), SCALE_RULE),
    ("exponential lam on an interval below 0",
     lambda: _one_prior("exponential", (Ref("w_interval__"),), "log", extra=[Var("w_interval__", "w", 1, "interval", (-1.0, 1.0))]),
     SCALE_RULE),
    ("studentt sigma -2", lambda: _one_prior("studentt", (3.0, 0.0, -2.0)), SCALE_RULE),
    ("lognormal sigma on an untransformed scalar", lambda: _one_prior("lognormal", (0.0, Ref("m")), "log"), SCALE_RULE),
    ("normal likelihood sigma -1", lambda: _one_lik("normal", [0.1, 0.2], sigma=-1.0), SCALE_RULE),
    ("normal likelihood sigma on an untransformed scalar", lambda: _one_lik("normal", [0.1, 0.2], sigma=Ref("m")), SCALE_RULE),
    ("studentt likelihood sigma 0", lambda: _one_lik("studentt", [0.1, 0.2], sigma=0.0, nu=3.0), SCALE_RULE),
    ("normal likelihood per-observation sigma with a negative",
     lambda: _one_lik("normal", [0.1, 0.2], sigma=np.array([1.0, -1.0])), "sigma must be a finite constant > 0 for every observation"),
    ("AR1 sigma on an untransformed scalar", lambda: _one_ar1(0.5, Ref("m")), SCALE_RULE),
    ("AR1 sigma -1", lambda: _one_ar1(0.5, -1.0), SCALE_RULE),
    ("poisson y = -1", lambda: _one_lik("poisson_log", [1.0, -1.0]), "poisson_log: y must be integers >= 0"),
    ("poisson y = 0.5", lambda: _one_lik("poisson_log", [1.0, 0.5]), "poisson_log: y must be integers >= 0"),
    ("bernoulli y = 2", lambda: _one_lik("bernoulli_logit", [1.0, 2.0]), "bernoulli_logit: y must be 0 or 1"),
    ("negative binomial alpha on an untransformed scalar", lambda: _one_lik("negative_binomial_log", [1.0, 2.0], alpha=Ref("m")),
     SCALE_RULE),
]


@pytest.mark.parametrize("what,model,msg", OUT_OF_SUPPORT, ids=[c[0] for c in OUT_OF_SUPPORT])
def test_validate_refuses_models_the_ir_cannot_keep_in_their_support(what, model, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        model().validate()


def test_validate_accepts_the_support_keeping_forms():
    for m in (_one_prior("halfnormal", (1.0,), "log"), _one_prior("halfnormal", (Ref("s_log__"),), "interval", (0.0, 3.0)),
              _one_prior("beta", (2.0, 2.0), "interval", (0.1, 1.0)), _one_prior("uniform", (0.0, 1.0), "interval", (0.25, 0.5)),
              _one_prior("normal", (Ref("m"), Ref("s_log__")), "log"), _one_prior("flat", ()),
              _one_lik("normal", [0.1, 0.2], sigma=np.array([1.0, 2.0])), _one_lik("studentt", [0.1, 0.2], sigma=Ref("s_log__"), nu=3.0),
              _one_lik("poisson_log", [0.0, 7.0]), _one_lik("bernoulli_logit", [0.0, 1.0]), _one_ar1(Ref("m"), Ref("s_log__")),
              _one_ar1(1.0, 0.3)):
        m.validate()


@pytest.mark.parametrize("rv_op,params", [("HalfNormalRV", (0.0, 1.0)), ("ExponentialRV", (0.5,)), ("UniformRV", (0.0, 1.0))])
def test_from_pymc_refuses_a_positive_variable_without_its_transform(fake_pytensor, rv_op, params):
    """pm.HalfNormal("sd", transform=None) and the like: the variable's own name is in the message."""
    from test_frontend_mock import Constant, FakeModel, bcast, elem, rv

    from pymc_b200 import from_pymc

    M = FakeModel("untransformed")
    mu = M.free(rv("NormalRV", "mu", Constant(0.0), Constant(1.0)), 1)
    sd = M.free(rv(rv_op, "sd", *[Constant(p) for p in params]), 1)
    M.observe(rv("NormalRV", "y", elem("Mul", bcast(mu), Constant(np.ones(3))), bcast(sd)), np.zeros(3))
    with pytest.raises(ValueError, match="on sd:"):
        from_pymc(M)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cid", CASE_IDS)
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid, monkeypatch):
    """Chain = warp, then the same handle with chain = CTA forced: each against the mp reference and the oracle, each
    bit-identical when repeated, the two equal to rounding.  Far-out interval points against the oracle."""
    from oracle import ir_numpy_families
    from pymc_b200 import engine

    m = build(cid)
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = ir_numpy_families.make_logp(m)
    Q, lp_mp, S, g_mp = mp_reference(cid)
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    far = far_interval_points(m)
    out = {}
    for team in ("warp", "cta"):
        if team == "cta":
            monkeypatch.setenv("B200_FORCE_TEAM", "1")
        lp, g = cm.logp_dlogp(Q)
        lp2, g2 = cm.logp_dlogp(Q)
        assert np.array_equal(lp, lp2) and np.array_equal(g, g2), (cid, team)
        assert_close_to_reference(lp, g, lp_mp, S, g_mp, (cid, team))
        assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12, (cid, team)
        assert np.max(np.abs(g - go) / np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))) <= 1e-12, (cid, team)
        out[team] = lp, g
        if far is not None:
            lpf, gf = cm.logp_dlogp(far)
            with np.errstate(all="ignore"):
                ref = [f(q) for q in far]
            for k, (a, b) in enumerate(ref):
                assert np.isfinite(lpf[k]) == np.isfinite(a), (cid, team, k)
                if np.isfinite(a):
                    assert abs(lpf[k] - a) <= 1e-12 * max(1.0, abs(a)), (cid, team, k)
                    fin = np.isfinite(b)
                    assert np.array_equal(np.isfinite(gf[k]), fin), (cid, team, k)
                    assert np.max(np.abs(gf[k][fin] - b[fin]), initial=0.0) <= 1e-12 * max(1.0, np.max(np.abs(b[fin]), initial=0.0))
    monkeypatch.delenv("B200_FORCE_TEAM")
    (lw, gw), (lc, gc) = out["warp"], out["cta"]
    assert np.all(np.abs(lw - lc) <= LP_TOL * S), cid
    assert np.all(np.max(np.abs(gw - gc), axis=1) <= GRAD_TOL * np.maximum(1.0, np.max(np.abs(gw), axis=1))), cid


BUCKET_NS = [32, 33, 64, 65, 128, 129, 192, 193, 256, 257, 512, 513, 1024, 1025, 2048, 2049, 3072, 3073, 4096]


def bucket(n):
    """(W, NPL) the dispatch gives an IR model of n coordinates: chain = warp up to 256, else chain = CTA of 8 warps."""
    if n <= 256:
        return 1, next(o for o in (1, 2, 4, 6, 8) if -(-n // 32) <= o)
    return 8, next(o for o in (2, 4, 8, 12, 16) if -(-n // 256) <= o)


def padded_model(n):
    """mu, log tau and n - 2 group effects a_j ~ Normal(mu, tau), one Normal observation of each."""
    rng = np.random.default_rng(n)
    G = n - 2
    idx = rng.permutation(G).astype(np.int32)
    return ModelIR(vars=[Var("mu", "mu", 1), Var("tau_log__", "tau", 1, "log"), Var("a", "a", G)],
                   priors=[Prior("normal", "mu", (0.0, 2.0)), Prior("halfnormal", "tau_log__", (1.0,)),
                           Prior("normal", "a", (Ref("mu"), Ref("tau_log__")))],
                   likelihoods=[Likelihood("normal", rng.standard_normal(G), [Term([("a", idx)])], sigma=0.7)])


def test_bucket_boundaries_reach_every_instantiation():
    """The (W, NPL) pair of each n in BUCKET_NS, by the rule of npl_warp / npl_team in csrc/b200nuts.cu: all ten
    instantiations of IrModel occur, and each n and n + 1 in the list sit on the two sides of a bucket boundary."""
    assert {bucket(n) for n in BUCKET_NS} == {(1, 1), (1, 2), (1, 4), (1, 6), (1, 8), (8, 2), (8, 4), (8, 8), (8, 12), (8, 16)}
    edges = [n for n in BUCKET_NS if n + 1 in BUCKET_NS]
    assert len(edges) == 9 and all(bucket(n) != bucket(n + 1) for n in edges)
    assert bucket(4096) == (8, 16)


@pytest.mark.gpu
def test_device_logp_at_the_bucket_boundaries():
    from oracle import ir_numpy
    from pymc_b200 import _lib, engine

    for n in BUCKET_NS:
        m = padded_model(n)
        assert m.n == n
        cm = engine.CompiledModel(m, specialise=False)
        f = ir_numpy.make_logp(m)
        Q = m.initial_point() + np.random.default_rng(n + 1).uniform(-1.0, 1.0, (5, n))
        lp, g = cm.logp_dlogp(Q)
        lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
        assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12, (n, bucket(n))
        assert np.max(np.abs(g - go) / np.max(np.abs(go), axis=1, keepdims=True)) <= 1e-12, (n, bucket(n))
    with pytest.raises(_lib.B200Error, match="exceeds the chain-per-CTA limit"):
        m = padded_model(4097)
        engine.CompiledModel(m, specialise=False).logp_dlogp(m.initial_point())


NUTS_CASES = [  # one per likelihood kind, two likelihoods, two AR(1) factors; fixed step sizes
    ("lik-normal-ref_log", 0.2), ("lik-studentt-nu4-ref_log", 0.2), ("lik-bernoulli", 0.3), ("lik-poisson", 0.1),
    ("lik-normal_logvar", 0.2), ("lik-binomial-obs-three_factors", 0.05), ("lik-negbin-ref_log-dominant_group", 0.1),
    ("lik-gamma-ref_log-offset_and_scalar_coef", 0.1), ("two_likelihoods-normal50-bernoulli20", 0.1), ("ar1-two", 0.1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("team", ["warp", "cta"])
@pytest.mark.parametrize("cid,eps", NUTS_CASES, ids=[c for c, _ in NUTS_CASES])
def test_fixed_step_nuts_matches_the_oracle_sampler(cid, eps, team, monkeypatch):
    from test_ir_families import _fixed_step_against_oracle

    if team == "cta":
        monkeypatch.setenv("B200_FORCE_TEAM", "1")
    _fixed_step_against_oracle(build(cid), eps, C=2, T=10)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle_on_two_likelihoods():
    from test_ir_families import _fixed_step_against_oracle

    m = build("two_likelihoods-normal50-bernoulli20")
    rng = np.random.default_rng(5)
    U = rng.standard_normal((m.n, 3)) * 0.05
    cov = np.diag(np.full(m.n, 0.05)) + U @ U.T
    _fixed_step_against_oracle(m, 0.25, dense_cov=0.5 * (cov + cov.T), C=2, T=10)


def _eta(m, L, q):
    """Linear predictor of likelihood L at one unconstrained point, in float64."""
    c, off, N = m.constrain(q), m.offsets(), len(L.y)
    x = q.copy()
    for v in m.vars:
        x[off[v.name] : off[v.name] + v.size] = np.ravel(c[v.rv_name])
    eta = np.zeros(N)
    for t in L.terms:
        term = np.ones(N) if t.coef is None else np.broadcast_to(np.asarray(t.coef, dtype=np.float64), (N,))
        for vn, idx in t.factors:
            v = m.var(vn)
            xv = x[off[v.name] : off[v.name] + v.size]
            term = term * (xv[idx] if idx is not None else (xv[0] if v.size == 1 else xv))
        eta = eta + term
    return eta, x


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [c for c in CASE_IDS if not c.startswith("prior-")] + ["prior-normal-none-c_c"])
def test_pointwise_log_likelihood_matches_scipy(cid):
    from pymc_b200 import engine

    m = build(cid)
    cm = engine.CompiledModel(m, specialise=False)
    Q = m.initial_point() + np.random.default_rng(8).uniform(-1.0, 1.0, (3, m.n))
    off = m.offsets()
    for lik, L in enumerate(m.likelihoods):
        ll = cm.pointwise_loglik(Q, lik=lik)
        assert ll.shape == (3, len(L.y))
        for k, q in enumerate(Q):
            eta, x = _eta(m, L, q)
            par = L.trials if L.dist == "binomial_logit" else (L.alpha if L.alpha is not None else L.sigma)
            s = x[off[m.var(par.var).name]] if isinstance(par, Ref) else (1.0 if par is None else np.asarray(par, dtype=np.float64))
            np.testing.assert_allclose(ll[k], scipy_loglik(L.dist, np.asarray(L.y), eta, s, L.nu), rtol=1e-12, atol=1e-12,
                                       err_msg=f"{cid} likelihood {lik}")


@pytest.mark.gpu
def test_model_create_refuses_tables_outside_the_support_through_the_c_abi():
    """b200_model_create makes the support checks of validate(), with the same words, for callers of the C ABI."""
    from test_ir_families import _create_raw

    def lowered(cid):
        low = ir.lower(build(cid))
        assert _create_raw(low) is None  # the unedited tables are accepted
        return low

    def var_index(cid, name):
        return [v.name for v in build(cid).vars].index(name)

    def param(low, k, a, kind, value, ref=-1):
        dist, var, ps = low.priors[k]
        ps = list(ps)
        ps[a] = (kind, value, ref)
        low.priors[k] = (dist, var, ps)

    edits = []

    def case(cid, msg):
        def reg(fn):
            edits.append((cid, fn, msg))
            return fn
        return reg

    @case("prior-halfnormal-log-c", "needs a log transform or an interval with lo >= 0")
    def _(low):
        low.vars[0, 2] = ir.TRANSFORMS[None]

    @case("prior-exponential-interval0_3-log", "needs a log transform or an interval with lo >= 0")
    def _(low):
        low.var_bounds[0] = (-1.0, 3.0)

    @case("prior-beta-interval0_1-c_c", "needs an interval inside [0, 1]")
    def _(low):
        low.var_bounds[0] = (0.0, 2.0)

    @case("prior-uniform-interval0_2-c_c", "needs an interval inside the Uniform bounds")
    def _(low):
        low.var_bounds[0] = (-2.0, 2.0)

    @case("prior-normal-none-c_c", SCALE_RULE)
    def _(low):
        param(low, 0, 1, 0, -1.0)

    @case("prior-cauchy-none-loc_log", SCALE_RULE)
    def _(low):
        param(low, 0, 1, 1, 0.0, int(low.vars[var_index("prior-cauchy-none-loc_log", "m"), 0]))  # beta = m: no transform

    @case("prior-halfcauchy-log-int", SCALE_RULE)
    def _(low):
        low.var_bounds[var_index("prior-halfcauchy-log-int", "w_interval__")] = (-1.0, 4.0)

    @case("lik-normal-const", SCALE_RULE)
    def _(low):
        low.liks[0]["sigma_value"] = -1.0

    @case("lik-studentt-nu4-ref_log", SCALE_RULE)
    def _(low):
        low.liks[0]["sigma_ref"] = 0  # b0: no transform

    @case("lik-normal-obs", "sigma must be a finite constant > 0 for every observation")
    def _(low):
        low.liks[0]["sigma_obs"] = low.liks[0]["sigma_obs"].copy()
        low.liks[0]["sigma_obs"][3] = -0.5

    @case("ar1-const", SCALE_RULE)
    def _(low):
        v, phi, sg, init = low.ar1[0]
        low.ar1[0] = (v, phi, (0, -1.0, -1), init)

    @case("ar1-ref-stochvol", SCALE_RULE)
    def _(low):
        v, phi, sg, init = low.ar1[0]
        low.ar1[0] = (v, phi, (1, 0.0, 0), init)  # mu: no transform

    @case("lik-poisson", "poisson_log: y must be integers >= 0")
    def _(low):
        low.liks[0]["y"] = low.liks[0]["y"].copy()
        low.liks[0]["y"][0] = -1.0

    @case("lik-poisson", "poisson_log: y must be integers >= 0")
    def _(low):
        low.liks[0]["y"] = low.liks[0]["y"].copy()
        low.liks[0]["y"][5] = 0.5

    @case("lik-bernoulli", "bernoulli_logit: y must be 0 or 1")
    def _(low):
        low.liks[0]["y"] = low.liks[0]["y"].copy()
        low.liks[0]["y"][2] = 2.0

    for cid, edit, msg in edits:
        low = lowered(cid)
        edit(low)
        err = _create_raw(low)
        assert err is not None and msg in err, (cid, msg, err)
