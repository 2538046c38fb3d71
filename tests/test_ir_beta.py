"""Beta regression likelihoods of the model IR (``ir.BETA_LIKS``): ``beta_logit``, y ~ Beta(mu = sigmoid(eta), nu = phi),
and ``beta_binomial_logit``, y ~ BetaBinomial(n, phi mu, phi (1 - mu)), with phi a constant or a scalar variable.

``_mp_logp`` writes the joint log-density with mpmath at 40 digits from the published definitions: the Beta density
lgamma(a + b) - lgamma(a) - lgamma(b) + (a - 1) log y + (b - 1) log(1 - y) and the BetaBinomial pmf binomln(n, y) +
lbeta(y + a, n - y + b) - lbeta(a, b), at a = phi mu, b = phi (1 - mu); the gradient is ``mpmath.diff``.  It reads the
``ModelIR`` dataclasses and nothing else of the package or of oracle/.  S = sum |additive pieces|: logp is compared to
1e-13 S; the gradient to 1e-12 max(1, |g|_inf) plus 1e-15 G, G the sum of the sizes of the parts d logp / d eta and
d logp / d phi are formed from (``_mp_grad_pieces``), as in tests/test_ir_survival.py.  Every BetaBinomial observation
with y <= 20 is also held to 1e-12 (|log f_i| + 1) on its own, which pins the cancellation-free small-count sums.

CPU: the reference against scipy.stats, the oracle (oracle/ir_numpy_beta.py) against the reference and central
differences on every catalogue case, the support rule through validate() and the C ABI, the lowered tables,
``specialise`` / ``fuse_design_columns``, and the sampler's data groups through the oracle-backed stand-in.  GPU: the
generic device function against both, the pointwise log-likelihood, fixed-step, lock-step and adaptive NUTS against the
oracle sampler."""
import ctypes
import zlib
from functools import lru_cache

import mpmath
import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import stats
from b200_helpers import (adaptive_against_oracle, fd_grad, fixed_step_against_oracle, logp_at_both_team_shapes,
                          random_dense_cov, refusal_after_edit)
from test_ir_bounded import _mp_constrain, _mp_eta, assert_close_to_reference
from test_ir_closed_set import MP_DPS

from pymc_b200 import _lib, ir
from pymc_b200.ir import Likelihood, ModelIR, Prior, Ref, Term, Var


# ------------------------------------------------------------------------------------------------------------------------
# the high-precision reference
# ------------------------------------------------------------------------------------------------------------------------
def _mp_ab(eta, phi):
    mu = 1 / (1 + mp.exp(-eta))
    return phi * mu, phi * (1 - mu)


def _mp_lik_pieces(dist, y, n, eta, phi):
    """Pieces of log p(y | eta) of one Beta / BetaBinomial observation (n: the trials, unused by the Beta)."""
    a, b = _mp_ab(eta, phi)
    if dist == "beta_logit":
        return [mp.loggamma(phi), -mp.loggamma(a), -mp.loggamma(b), (a - 1) * mp.log(y), (b - 1) * mp.log(1 - y)]
    return [mp.loggamma(n + 1), -mp.loggamma(y + 1), -mp.loggamma(n - y + 1), mp.loggamma(y + a), -mp.loggamma(a),
            mp.loggamma(n - y + b), -mp.loggamma(b), -mp.loggamma(n + phi), mp.loggamma(phi)]


def _mp_phi(m, L, x):
    return x[m.var(L.phi.var).name][0] if isinstance(L.phi, Ref) else mpf(float(L.phi))


def _mp_trials(L):
    N = len(L.y)
    return [mpf(0)] * N if L.trials is None else [mpf(float(v)) for v in np.broadcast_to(L.trials, (N,))]


def _mp_prior(p, x, vn, par):
    a = [par(t, x) for t in p.params]
    if p.dist == "normal":
        return [t for xi in x[vn] for t in (-((xi - a[0]) / a[1]) ** 2 / 2, -mp.log(a[1]), -mp.log(2 * mp.pi) / 2)]
    if p.dist == "halfnormal":
        return [t for xi in x[vn] for t in (-(xi / a[0]) ** 2 / 2, -mp.log(a[0]), mp.log(2) / 2 - mp.log(mp.pi) / 2)]
    if p.dist == "gamma":
        return [t for xi in x[vn] for t in ((a[0] - 1) * mp.log(xi), -a[1] * xi, a[0] * mp.log(a[1]), -mp.loggamma(a[0]))]
    assert p.dist == "uniform"
    return [-mp.log(a[1] - a[0]) for _ in x[vn]]


def _mp_factors(m):
    name = lambda r: m.var(r).name  # noqa: E731
    par = lambda a, x: x[name(a.var)][0] if isinstance(a, Ref) else mpf(float(a))  # noqa: E731
    out = []
    for p in m.priors:
        vn = name(p.var)
        out.append(({vn} | {name(a.var) for a in p.params if isinstance(a, Ref)},
                    lambda x, p=p, vn=vn: _mp_prior(p, x, vn, par)))
    for L in m.likelihoods:
        N = len(L.y)
        y = [mpf(float(v)) for v in L.y]
        deps = {name(vn) for t in L.terms for vn, _ in t.factors}
        for s in (L.phi, L.sigma):
            if isinstance(s, Ref):
                deps.add(name(s.var))
        if L.dist == "normal":  # an older factor beside the Beta ones
            def lik(x, L=L, y=y, N=N):
                eta, s = _mp_eta(m, L, x), par(L.sigma, x)
                return [t for i in range(N) for t in (-((y[i] - eta[i]) / s) ** 2 / 2, -mp.log(s), -mp.log(2 * mp.pi) / 2)]
        else:
            def lik(x, L=L, y=y, N=N, n=_mp_trials(L)):
                eta, phi = _mp_eta(m, L, x), _mp_phi(m, L, x)
                return [t for i in range(N) for t in _mp_lik_pieces(L.dist, y[i], n[i], eta[i], phi)]
        out.append((deps, lik))
    return out


def _mp_logp(m, q):
    with mp.workdps(MP_DPS):
        x, jac = _mp_constrain(m, [mpf(float(t)) for t in q])
        pieces = [t for j in jac for t in j] + [t for _, f in _mp_factors(m) for t in f(x)]
        return float(mp.fsum(pieces)), float(mp.fsum(abs(t) for t in pieces))


def _mp_grad(m, q):
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


def _mp_loglik(m, L, q):
    """log f_i of every observation of Beta likelihood L at q."""
    with mp.workdps(MP_DPS):
        x, _ = _mp_constrain(m, [mpf(float(t)) for t in q])
        eta, phi, n = _mp_eta(m, L, x), _mp_phi(m, L, x), _mp_trials(L)
        return np.array([float(mp.fsum(_mp_lik_pieces(L.dist, mpf(float(L.y[i])), n[i], eta[i], phi)))
                         for i in range(len(L.y))])


def _mp_grad_pieces(m, q):
    """G = the sum over observations of the sizes of the parts d logp / d eta and d logp / d phi are formed from:
    (1 + phi mu (1 - mu) + phi) (1 + |log y| + |log(1 - y)| + |psi| of a, b, phi and, for the BetaBinomial, of y + a,
    n - y + b and n + phi); the factor phi is that of the chain rule through a log transform."""
    with mp.workdps(MP_DPS):
        x, _ = _mp_constrain(m, [mpf(float(t)) for t in q])
        G = mpf(0)
        for L in m.likelihoods:
            eta = _mp_eta(m, L, x)
            if L.dist == "normal":
                s = mpf(float(L.sigma))
                G += sum((1 + abs((mpf(float(L.y[i])) - eta[i]) / s)) / s for i in range(len(L.y)))
                continue
            phi, n = _mp_phi(m, L, x), _mp_trials(L)
            for i in range(len(L.y)):
                y = mpf(float(L.y[i]))
                a, b = _mp_ab(eta[i], phi)
                w = phi * (a / phi) * (b / phi)
                parts = 1 + abs(mp.digamma(a)) + abs(mp.digamma(b)) + abs(mp.digamma(phi))
                if L.dist == "beta_logit":
                    parts += abs(mp.log(y)) + abs(mp.log(1 - y))
                else:
                    parts += abs(mp.digamma(y + a)) + abs(mp.digamma(n[i] - y + b)) + abs(mp.digamma(n[i] + phi))
                G += (1 + w + phi) * parts
        return float(G)


# ------------------------------------------------------------------------------------------------------------------------
# the case catalogue
# ------------------------------------------------------------------------------------------------------------------------
def _phi_vars(kind, phi0=8.0):
    if kind == "ref_log":
        return [Var("phi_log__", "phi", 1, "log", initial=np.log(phi0))], [Prior("gamma", "phi_log__", (2.0, 0.1))], \
            Ref("phi_log__")
    if kind == "ref_int":
        return [Var("phi_interval__", "phi", 1, "interval", (0.02, 50.0))], \
            [Prior("uniform", "phi_interval__", (0.02, 50.0))], Ref("phi_interval__")
    return [], [], phi0


def _regression_case(dist, kind, shape, rng, N=12):
    """b0 + b1 x (or a design term and a group effect) under a Beta / BetaBinomial likelihood."""
    x = rng.standard_normal(N)
    eta = 0.3 + 0.8 * x
    mu = 1.0 / (1.0 + np.exp(-eta))
    vars_ = [Var("b0", "b0", 1), Var("b1", "b1", 1)]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "b1", (0.0, 1.0))]
    terms = [Term([("b0", None)]), Term([("b1", None)], coef=x)]
    if shape == "design":
        X = np.column_stack([np.ones(N), x, rng.standard_normal(N)])
        vars_ = [Var("beta", "beta", 3), Var("g", "g", 3)]
        priors = [Prior("normal", "beta", (0.0, 1.5)), Prior("normal", "g", (0.0, 1.0))]
        terms = [Term([("beta", None)], coef=X), Term([("g", np.arange(N, dtype=np.int32) % 3)])]
    pv, pp, phi = _phi_vars(kind)
    p = rng.beta(mu * 8.0, (1.0 - mu) * 8.0)
    if dist == "beta_logit":
        return ModelIR(vars=vars_ + pv, priors=priors + pp, likelihoods=[Likelihood(dist, p, terms, phi=phi)])
    trials = 12.0 if shape != "obs_trials" else rng.integers(0, 50, N).astype(np.float64)
    y = rng.binomial(np.asarray(trials, dtype=np.int64), p).astype(np.float64)
    if shape == "obs_trials":  # y = 0, y = n, n = 0 and n = 1 among them
        trials[:4] = [0.0, 1.0, 7.0, 9.0]
        y[:4] = [0.0, 1.0, 0.0, 9.0]
    return ModelIR(vars=vars_ + pv, priors=priors + pp, likelihoods=[Likelihood(dist, y, terms, trials=trials, phi=phi)])


def _edge_case(dist, phi, kind="const"):
    """eta = b0 + an offset from -30 to 30; the Beta's y from 1e-12 to 1 - 1e-12, the BetaBinomial's small counts (n <= 30,
    so every bracket is a short sum whatever a and b are) with y = 0 and y = n."""
    off = np.array([-30.0, 30.0, -3.0, 0.0, 2.0, 30.0, -30.0, 0.5])
    N = len(off)
    pv, pp, ph = _phi_vars(kind, phi)
    terms = [Term([("b0", None)]), Term([], coef=off)]
    vars_, priors = [Var("b0", "b0", 1)] + pv, [Prior("normal", "b0", (0.0, 1.0))] + pp
    if dist == "beta_logit":
        y = np.array([1e-12, 1.0 - 1e-12, 0.02, 0.5, 0.97, 1e-12, 1.0 - 1e-12, 0.3])
        return ModelIR(vars=vars_, priors=priors, likelihoods=[Likelihood(dist, y, terms, phi=ph)])
    n = np.array([30.0, 30.0, 10.0, 1.0, 20.0, 0.0, 5.0, 25.0])
    y = np.array([0.0, 30.0, 3.0, 1.0, 20.0, 0.0, 5.0, 12.0])
    assert N == len(y)
    return ModelIR(vars=vars_, priors=priors, likelihoods=[Likelihood(dist, y, terms, trials=n, phi=ph)])


def _large_count_case(phi):
    """n = 1000 with y = 500, and neighbours across the sum / lgamma cutoff."""
    n = np.array([1000.0, 1000.0, 1000.0, 40.0, 31.0, 32.0, 33.0, 200.0])
    y = np.array([500.0, 3.0, 990.0, 33.0, 31.0, 0.0, 1.0, 150.0])
    off = np.linspace(-1.5, 1.5, len(y))
    return ModelIR(vars=[Var("b0", "b0", 1)], priors=[Prior("normal", "b0", (0.0, 1.0))],
                   likelihoods=[Likelihood("beta_binomial_logit", y, [Term([("b0", None)]), Term([], coef=off)],
                                           trials=n, phi=phi)])


def _mixed_case(rng):
    """A Beta and a BetaBinomial likelihood with an older one (Normal) on shared coefficients."""
    a = _regression_case("beta_logit", "ref_log", "plain", rng, N=8)
    b = _regression_case("beta_binomial_logit", "const", "obs_trials", rng, N=8)
    x = rng.standard_normal(6)
    Lb, Ln = b.likelihoods[0], Likelihood("normal", rng.standard_normal(6), [Term([("b0", None)]), Term([("b1", None)], coef=x)],
                                          sigma=1.3)
    Lb.name, Ln.name = "y2", "y3"
    return ModelIR(vars=a.vars, priors=a.priors, likelihoods=a.likelihoods + [Lb, Ln])


CASES = {}
for _d in ir.BETA_LIKS:
    _shapes = ("plain", "design", "again") if _d == "beta_logit" else ("plain", "design", "obs_trials")
    for _j, _sh in enumerate(_shapes):
        _k = ("const", "ref_log", "ref_int")[_j]
        CASES[f"{_d}-{_sh}-{_k}"] = (lambda rng, d=_d, k=_k, sh=_sh: _regression_case(d, k, sh, rng))
    for _p in (0.05, 1.0, 1e3, 1e6) + ((1e8,) if _d == "beta_binomial_logit" else ()):
        CASES[f"{_d}-edges-phi{_p:g}"] = (lambda rng, d=_d, p=_p: _edge_case(d, p))
    CASES[f"{_d}-edges-ref"] = (lambda rng, d=_d: _edge_case(d, 1e3, "ref_log"))
for _p in (0.5, 50.0):
    CASES[f"beta_binomial_logit-large-phi{_p:g}"] = (lambda rng, p=_p: _large_count_case(p))
CASES["mixed"] = _mixed_case
CASE_IDS = list(CASES)


def build(cid):
    return CASES[cid](np.random.default_rng(zlib.crc32(cid.encode())))


def points(m, cid):
    """The initial point + U(-0.5, 0.5), twice."""
    rng = np.random.default_rng(zlib.crc32(cid.encode()) + 1)
    q0 = m.initial_point()
    return np.array([q0 + rng.uniform(-0.5, 0.5, m.n) for _ in range(2)])


@lru_cache(maxsize=None)
def mp_reference(cid):
    m = build(cid)
    Q = points(m, cid)
    lp, S = np.array([_mp_logp(m, q) for q in Q]).T
    return Q, lp, S, np.array([_mp_grad(m, q) for q in Q]), np.array([_mp_grad_pieces(m, q) for q in Q])


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference and the oracle
# ------------------------------------------------------------------------------------------------------------------------
def _mp_one(dist, y, eta, phi, n=0.0):
    with mp.workdps(MP_DPS):
        return float(mp.fsum(_mp_lik_pieces(dist, mpf(y), mpf(n), mpf(eta), mpf(phi))))


def test_mp_pieces_equal_scipy():
    """Beta.logpdf and betabinom.logpmf at a = phi sigmoid(eta), b = phi sigmoid(-eta)."""
    for y, eta, phi in [(0.3, 0.0, 2.0), (0.01, -1.5, 10.0), (0.95, 2.0, 0.7), (0.5, 0.4, 300.0), (1e-6, -3.0, 1.0)]:
        mu = 1.0 / (1.0 + np.exp(-eta))
        want = stats.beta.logpdf(y, mu * phi, (1.0 - mu) * phi)
        got = _mp_one("beta_logit", y, eta, phi)
        assert abs(got - want) <= 1e-11 * max(1.0, abs(want)), (y, eta, phi, got, want)
    for y, n, eta, phi in [(3, 10, 0.0, 2.0), (0, 5, 1.0, 0.5), (7, 7, -0.5, 30.0), (500, 1000, 0.2, 4.0), (1, 1, 0.0, 1.0),
                           (12, 40, -1.0, 1e4)]:
        mu = 1.0 / (1.0 + np.exp(-eta))
        want = stats.betabinom.logpmf(y, n, mu * phi, (1.0 - mu) * phi)
        got = _mp_one("beta_binomial_logit", y, eta, phi, n)
        assert abs(got - want) <= 1e-10 * max(1.0, abs(want)), (y, n, eta, phi, got, want)


def test_the_catalogue_covers_the_beta_forms():
    seen = set()
    for cid in CASE_IDS:
        m = build(cid)
        m.validate()
        for L in m.likelihoods:
            if L.dist not in ir.BETA_LIKS:
                seen.add("older")
                continue
            seen.add((L.dist, "ref" if isinstance(L.phi, Ref) else "const"))
            if not isinstance(L.phi, Ref):
                seen.add((L.dist, "phi", float(L.phi)))
            seen.add((L.dist, "design")) if any(ir.is_design(t) for t in L.terms) else None
            eta_off = [t.coef for t in L.terms if not t.factors]
            if eta_off and np.min(eta_off[0]) == -30.0 and np.max(eta_off[0]) == 30.0:
                seen.add((L.dist, "eta30"))
            if L.dist == "beta_logit":
                if np.min(L.y) == 1e-12 and np.max(L.y) == 1.0 - 1e-12:
                    seen.add("y_edges")
                continue
            n = np.broadcast_to(L.trials, L.y.shape)
            seen.add(("trials", "obs" if np.ndim(L.trials) == 1 else "const"))
            seen |= {s for s, ok in (("y=0", np.any(L.y == 0)), ("y=n", np.any((L.y == n) & (n > 0))), ("n=0", np.any(n == 0)),
                                     ("n=1", np.any(n == 1)), ("n=1000,y=500", np.any((n == 1000) & (L.y == 500)))) if ok}
        if len(m.likelihoods) > 1 and "older" in seen:
            seen.add("mixed")
    for d in ir.BETA_LIKS:
        assert {(d, "ref"), (d, "const"), (d, "design"), (d, "eta30")} <= seen, d
        assert {(d, "phi", p) for p in (0.05, 1e6)} <= seen, d
    assert ("beta_binomial_logit", "phi", 1e8) in seen
    assert {"y_edges", ("trials", "obs"), ("trials", "const"), "y=0", "y=n", "n=0", "n=1", "n=1000,y=500", "mixed"} <= seen


@pytest.mark.parametrize("cid", CASE_IDS)
def test_oracle_matches_the_mp_reference_and_central_differences(cid):
    from oracle import ir_numpy_beta

    m = build(cid)
    f = ir_numpy_beta.make_logp(m)
    Q, lp_mp, S, g_mp, G = mp_reference(cid)
    lp, g = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    assert np.all(np.isfinite(lp)) and np.all(np.isfinite(g)), cid
    assert_close_to_reference(lp, g, lp_mp, S, g_mp, G, cid)
    gf = fd_grad(f, Q[0], h=1e-6)
    assert np.max(np.abs(gf - g[0])) <= 1e-5 * max(1.0, np.max(np.abs(g[0]))), cid


def _small_counts_within(loglik, cid, q):
    """Every BetaBinomial observation with y <= 20 of case cid within 1e-12 (|log f_i| + 1) of the reference."""
    m = build(cid)
    checked = 0
    for k, L in enumerate(m.likelihoods):
        if L.dist != "beta_binomial_logit":
            continue
        want = _mp_loglik(m, L, q)
        got = loglik(k, L)
        small = L.y <= 20
        err = np.abs(got - want)[small]
        assert np.all(err <= 1e-12 * (np.abs(want[small]) + 1.0)), (cid, err, want[small])
        checked += int(small.sum())
    return checked


def test_small_counts_keep_their_digits_at_every_phi():
    from oracle import ir_numpy_beta

    checked = 0
    for cid in CASE_IDS:
        m = build(cid)
        if not any(L.dist == "beta_binomial_logit" for L in m.likelihoods):
            continue
        f = ir_numpy_beta.make_logp(m)
        for q in points(m, cid):
            x, _ = f.constrained(q)
            checked += _small_counts_within(lambda k, L: f.loglik(L, x), cid, q)
    assert checked > 100
    # a and b of 1e8 and more are among them
    m = build("beta_binomial_logit-edges-phi1e+08")
    assert float(m.likelihoods[0].phi) == 1e8


def scipy_pointwise(L, eta, phi):
    mu = 1.0 / (1.0 + np.exp(-eta))
    if L.dist == "beta_logit":
        return stats.beta.logpdf(L.y, mu * phi, (1.0 - mu) * phi)
    return stats.betabinom.logpmf(L.y, np.broadcast_to(L.trials, L.y.shape), mu * phi, (1.0 - mu) * phi)


SCIPY_BUILDS = [("beta", "var"), ("beta", "const"), ("beta_binomial", "var"), ("beta_binomial", "const")]


def test_oracle_pointwise_equals_scipy_on_the_builders():
    from oracle import ir_numpy_beta

    for dist, phi in SCIPY_BUILDS:
        m = ir.beta_regression_ir(dist, phi, n_obs=80)
        f = ir_numpy_beta.make_logp(m)
        q = m.initial_point() + np.random.default_rng(2).uniform(-0.5, 0.5, m.n)
        x, _ = f.constrained(q)
        L = m.likelihoods[0]
        want = scipy_pointwise(L, f.eta(L, x)[0], f.param(L, x)[0])
        np.testing.assert_allclose(f.loglik(L, x), want, rtol=1e-11, atol=1e-11, err_msg=f"{dist} {phi}")


def test_the_oracle_covers_models_that_mix_old_and_new_factors():
    from oracle import ir_numpy_beta, ir_numpy_mixture

    a, b = ir.beta_regression_ir("beta", "var", n_obs=50), ir.mixture_ir("poisson", K=2, weights="const", n_obs=40)
    L2 = b.likelihoods[0]
    L2.name = "y2"
    m = ModelIR(vars=a.vars + b.vars, priors=a.priors + b.priors, likelihoods=a.likelihoods + [L2])
    f = ir_numpy_beta.make_logp(m)
    q = m.initial_point() + np.random.default_rng(5).uniform(-0.3, 0.3, m.n)
    lp, g = f(q)
    x, _ = f.constrained(q)
    want = float(np.sum(f.loglik(m.likelihoods[0], x))) + ir_numpy_mixture.make_logp(
        ModelIR(vars=m.vars, priors=m.priors, likelihoods=[L2]))(q)[0]
    assert abs(lp - want) <= 1e-12 * abs(want)
    assert np.max(np.abs(fd_grad(f, q) - g)) <= 1e-5 * max(1.0, np.max(np.abs(g)))


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the support rule, lowering, specialise, fuse_design_columns, the sampler's data groups
# ------------------------------------------------------------------------------------------------------------------------
def _one(dist, y, **kw):
    kw.setdefault("phi", 5.0)
    if dist == "beta_binomial_logit":
        kw.setdefault("trials", 10.0)
    return ModelIR(vars=[Var("b", "b", 1), Var("s_log__", "s", 1, "log")],
                   likelihoods=[Likelihood(dist, np.asarray(y, dtype=np.float64), [Term([("b", None)])], **kw)])


REFUSALS = [  # (what, dist, y, slots, the words validate() and b200_model_create share)
    ("y_zero", "beta_logit", [0.5, 0.0], {}, ir.BETA_Y),
    ("y_one", "beta_logit", [1.0, 0.5], {}, ir.BETA_Y),
    ("y_nan", "beta_logit", [0.5, np.nan], {}, ir.BETA_Y),
    ("y_above_one", "beta_logit", [0.5, 2.0], {}, ir.BETA_Y),
    ("trials_negative", "beta_binomial_logit", [1.0, 0.0], {"trials": np.array([3.0, -1.0])}, ir.BB_TRIALS),
    ("trials_fraction", "beta_binomial_logit", [1.0, 0.0], {"trials": 2.5}, ir.BB_TRIALS),
    ("trials_inf", "beta_binomial_logit", [1.0, 0.0], {"trials": np.inf}, ir.BB_TRIALS),
    ("y_above_trials", "beta_binomial_logit", [1.0, 11.0], {}, ir.ZIB_Y),
    ("y_negative", "beta_binomial_logit", [-1.0, 1.0], {}, ir.ZIB_Y),
    ("y_fraction", "beta_binomial_logit", [1.5, 1.0], {}, ir.ZIB_Y),
    ("phi_zero", "beta_logit", [0.5], {"phi": 0.0}, "phi must be a finite constant > 0"),
    ("phi_inf", "beta_binomial_logit", [1.0], {"phi": np.inf}, "phi must be a finite constant > 0"),
    ("phi_not_positive_support", "beta_logit", [0.5], {"phi": Ref("b")}, "positive support"),
    ("phi_missing", "beta_binomial_logit", [1.0], {"phi": None}, "beta_binomial_logit needs phi"),
    ("phi_per_observation", "beta_logit", [0.5, 0.5], {"phi": np.ones(2)}, "phi must be one constant or a scalar variable"),
    ("sigma", "beta_logit", [0.5], {"sigma": 1.0}, ir.BETA_SLOTS),
    ("alpha", "beta_binomial_logit", [1.0], {"alpha": 1.0}, ir.BETA_SLOTS),
    ("lower", "beta_logit", [0.5], {"lower": 0.1}, ir.BETA_SLOTS),
    ("upper", "beta_binomial_logit", [1.0], {"upper": 5.0}, ir.BETA_SLOTS),
    ("cutpoints", "beta_logit", [0.5], {"cutpoints": np.array([0.0, 1.0])}, ir.BETA_SLOTS),
    ("psi", "beta_binomial_logit", [1.0], {"psi": 0.5}, ir.BETA_SLOTS),
    ("weights", "beta_logit", [0.5], {"weights": np.array([0.5, 0.5])}, ir.BETA_SLOTS),
    ("components", "beta_logit", [0.5], {"components": np.array([0.5, 0.5])}, ir.BETA_SLOTS),
    ("trials_on_beta", "beta_logit", [0.5], {"trials": 3.0}, ir.BETA_TRIALS),
]


@pytest.mark.parametrize("what,dist,y,slots,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_validate_refuses_each_clause_of_the_support_rule(what, dist, y, slots, msg):
    with pytest.raises(ValueError) as e:
        _one(dist, y, **slots).validate()
    assert msg in str(e.value), (what, str(e.value))


def test_validate_accepts_the_rule_and_keeps_the_other_refusals():
    _one("beta_logit", [1e-300, 1.0 - 2 ** -53]).validate()
    _one("beta_binomial_logit", [0.0, 10.0]).validate()
    _one("beta_binomial_logit", [0.0, 0.0, 3.0], trials=np.array([0.0, 1.0, 3.0])).validate()
    _one("beta_logit", [0.5], phi=Ref("s_log__")).validate()
    with pytest.raises(ValueError, match="phi belongs to the beta_logit / beta_binomial_logit likelihoods"):
        ModelIR(vars=[Var("b", "b", 1)], likelihoods=[Likelihood("normal", np.ones(2), [Term([("b", None)])], sigma=1.0,
                                                                 phi=2.0)]).validate()
    with pytest.raises(ValueError, match="trials belong to binomial_logit"):  # the older words stay
        ModelIR(vars=[Var("b", "b", 1)], likelihoods=[Likelihood("poisson_log", np.ones(2), [Term([("b", None)])],
                                                                 trials=3.0)]).validate()
    with pytest.raises(ValueError, match="prior 'beta_binomial' is not in the closed set"):
        ModelIR(vars=[Var("b", "b", 1)], priors=[Prior("beta_binomial", "b", (1.0, 1.0))]).validate()


def test_lowered_tables_hold_the_dist_the_y_block_and_the_slot():
    for dist, phi, want in (("beta", "var", 26), ("beta", "const", 26), ("beta_binomial", "var", 27),
                            ("beta_binomial", "const", 27)):
        m = ir.beta_regression_ir(dist, phi, n_obs=40)
        L = m.likelihoods[0]
        N = len(L.y)
        c_ir, keep = _lib.build_ir(ir.lower(m))
        lik = ctypes.cast(c_ir.liks, ctypes.POINTER(_lib.IrLik))[0]
        assert lik.dist == want == ir.LIK_DISTS[L.dist] and lik.N == N and lik.y_var == 0 and lik.nu == 0.0
        rows = 2 if dist == "beta_binomial" else 1
        block = np.ctypeslib.as_array(ctypes.cast(lik.y, ctypes.POINTER(ctypes.c_double)), (rows, N))
        assert np.array_equal(block[0], L.y)
        if rows == 2:
            assert np.array_equal(block[1], L.trials)
        if phi == "var":
            assert lik.sigma_kind == ir.SIGMA_REF and lik.sigma.kind == 1 and lik.sigma.ref == m.offsets()["phi_log__"]
        else:
            assert lik.sigma_kind == ir.SIGMA_CONST and lik.sigma.value == float(L.phi)
    low = ir.lower(_one("beta_binomial_logit", [1.0, 4.0], trials=7.0))
    assert np.array_equal(low.liks[0]["y"], [[1.0, 4.0], [7.0, 7.0]])  # constant trials fill the second row


def test_the_example_builder():
    m = ir.beta_regression_ir("beta", "var")
    L = m.likelihoods[0]
    assert L.dist == "beta_logit" and isinstance(L.phi, Ref) and np.all((L.y > 0) & (L.y < 1)) and L.trials is None
    assert ir.beta_regression_ir("beta", "const").likelihoods[0].phi == 15.0
    m = ir.beta_regression_ir("beta_binomial", "var", n_obs=2000)
    L = m.likelihoods[0]
    assert L.dist == "beta_binomial_logit" and np.ndim(L.trials) == 1 and len(np.unique(L.trials)) > 20
    # overdispersion: the spread of y / n about its mean is well above the Binomial's
    p = L.y / L.trials
    binom_var = np.mean(p * (1 - p) / L.trials)
    assert np.var(p) > 2.0 * binom_var
    with pytest.raises(ValueError):
        ir.beta_regression_ir("gamma")
    with pytest.raises(ValueError):
        ir.beta_regression_ir("beta", "random")


def _as_columns(m):
    """The builders' design term written one column per term, the form from_pymc produces for dot(X, beta)."""
    import copy

    out = copy.deepcopy(m)
    for L in out.likelihoods:
        terms = []
        for t in L.terms:
            if ir.is_design(t):
                X = np.asarray(t.coef)
                terms += [Term([(t.factors[0][0], np.full(len(L.y), k, dtype=np.int32))], coef=X[:, k].copy())
                          for k in range(X.shape[1])]
            else:
                terms.append(t)
        L.terms = terms
    return out


def test_specialise_declines_and_fuse_design_columns_keeps_the_y_block():
    from oracle import ir_numpy_beta

    for dist, phi in SCIPY_BUILDS:
        m = ir.beta_regression_ir(dist, phi, n_obs=60)
        assert ir.specialise(m) is None and ir.specialise(m, extended=True) is None
        cols = _as_columns(m)
        fused = ir.fuse_design_columns(cols)
        L, F = m.likelihoods[0], fused.likelihoods[0]
        assert F.dist == L.dist and np.array_equal(F.y, L.y) and sum(ir.is_design(t) for t in F.terms) == 1
        assert F.phi == L.phi and ((F.trials is None and L.trials is None) or np.array_equal(F.trials, L.trials))
        assert np.array_equal(ir.lower(fused).liks[0]["y"], ir.lower(m).liks[0]["y"])
        f, g = ir_numpy_beta.make_logp(fused), ir_numpy_beta.make_logp(cols)
        q = m.initial_point() + np.random.default_rng(3).uniform(-0.5, 0.5, m.n)
        (a, ga), (b, gb) = f(q), g(q)
        assert abs(a - b) <= 1e-12 * abs(b) and np.allclose(ga, gb, rtol=1e-11, atol=1e-11)


def test_sampler_records_the_data_and_the_beta_log_likelihood():
    """The sampler on the oracle-backed stand-in: observed_data keeps y, constant_data the per-observation trials, and
    the log_likelihood group holds betabinom.logpmf of every observation."""
    from b200_helpers import OracleEngine
    from oracle import ir_numpy_beta
    from pymc_b200 import engine, sampling

    m = ir.beta_regression_ir("beta_binomial", "var", n_obs=60, n_groups=4, seed=5)

    class IrStandIn(OracleEngine):
        def __init__(self, model):
            self.ir, self.spec = model, engine._ir_spec(model)
            self.n, self.f = model.n, ir_numpy_beta.make_logp(model)

        def pointwise_loglik(self, draws, lik=0):
            q = np.asarray(draws)
            L = self.ir.likelihoods[lik]
            out = np.empty(q.shape[:-1] + (len(L.y),))
            for ix in np.ndindex(*q.shape[:-1]):
                out[ix] = self.f.loglik(L, self.f.constrained(q[ix])[0])
            return out

    res = sampling.sample_b200_nuts(5, tune=10, chains=2, random_seed=4, model=IrStandIn(m), momentum="numpy",
                                    keep_untransformed=True, idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
    L = m.likelihoods[0]
    assert np.array_equal(res.constant_data["y_trials"], L.trials)
    assert np.array_equal(res.observed_data["y"], L.y)
    ll = res.log_likelihood["y"]
    assert ll.shape == (2, 5, 60)
    X = L.terms[2].coef
    g = L.terms[1].factors[1][1]
    for c in range(2):
        for d in range(5):
            P = {k: res.posterior[k][c, d] for k in ("b0", "z", "sigma_a", "beta", "phi")}
            eta = P["b0"] + P["sigma_a"] * P["z"][g] + X @ P["beta"]
            np.testing.assert_allclose(ll[c, d], scipy_pointwise(L, eta, P["phi"]), rtol=1e-11, atol=1e-11)


def test_model_create_refuses_malformed_beta_tables_through_the_c_abi():
    """prepare_ir makes the checks of validate(), with the same words, for callers of the C ABI; a Beta likelihood is not
    a latent factor."""
    def set_y(row, k, value):
        def edit(low):
            y = low.liks[0]["y"].copy()
            if y.ndim == 1:
                y[k] = value
            else:
                y[row, k] = value
            low.liks[0]["y"] = y
        return edit

    beta = lambda phi="var": (lambda: ir.beta_regression_ir("beta", phi, n_obs=30))  # noqa: E731
    bb = lambda phi="var": (lambda: ir.beta_regression_ir("beta_binomial", phi, n_obs=30))  # noqa: E731
    bad_phi = lambda low: low.liks[0].update(sigma_value=-1.0, sigma_kind=ir.SIGMA_CONST)  # noqa: E731
    obs_phi = lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_OBS, sigma_obs=np.ones(30))  # noqa: E731
    no_phi = lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_NONE)  # noqa: E731
    with_nu = lambda low: low.liks[0].update(nu=3.0)  # noqa: E731
    as_latent = lambda low: low.liks[0].update(y_var=1)  # noqa: E731
    cases = [
        (beta(), set_y(0, 0, 0.0), ir.BETA_Y), (beta("const"), set_y(0, 3, 1.0), ir.BETA_Y),
        (beta(), set_y(0, 5, np.nan), ir.BETA_Y),
        (bb(), set_y(1, 0, -1.0), ir.BB_TRIALS), (bb("const"), set_y(1, 2, 4.5), ir.BB_TRIALS),
        (bb(), set_y(1, 2, np.inf), ir.BB_TRIALS),
        (bb(), set_y(0, 0, 1e6), ir.ZIB_Y), (bb("const"), set_y(0, 1, -1.0), ir.ZIB_Y), (bb(), set_y(0, 1, 0.5), ir.ZIB_Y),
        (beta(), bad_phi, "phi must be a finite constant > 0"), (bb(), bad_phi, "phi must be a finite constant > 0"),
        (beta(), obs_phi, "phi must be a constant or a scalar variable"),
        (bb(), no_phi, "phi must be a constant or a scalar variable"),
        (beta(), with_nu, ir.BETA_SLOTS), (bb(), with_nu, ir.BETA_SLOTS),
        (beta(), as_latent, "latent factor"), (bb(), as_latent, "latent factor"),
    ]
    for builder, edit, msg in cases:
        err = refusal_after_edit(builder, edit)
        assert err is not None and msg in err, (msg, err)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
BUILDERS = {
    "beta_var": lambda: ir.beta_regression_ir("beta", "var"),                                       # n = 13: warp
    "beta_var_cta": lambda: ir.beta_regression_ir("beta", "var", n_obs=1500, n_groups=300, seed=7),  # n = 305: CTA
    "beta_const": lambda: ir.beta_regression_ir("beta", "const"),
    "beta_binomial_var": lambda: ir.beta_regression_ir("beta_binomial", "var"),
    "beta_binomial_var_cta": lambda: ir.beta_regression_ir("beta_binomial", "var", n_obs=1200, n_groups=280, seed=8),
    "beta_binomial_const": lambda: ir.beta_regression_ir("beta_binomial", "const"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("cid", CASE_IDS)
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid):
    """Chain = warp, then chain = CTA forced: each against the mp reference and the oracle, bit-identical when repeated."""
    from oracle import ir_numpy_beta
    from pymc_b200 import engine

    m = build(cid)
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = ir_numpy_beta.make_logp(m)
    Q, lp_mp, S, g_mp, G = mp_reference(cid)
    go = np.array([f(q)[1] for q in Q])
    lo = np.array([f(q)[0] for q in Q])
    for team, (lp, g) in logp_at_both_team_shapes(cm, Q).items():
        assert np.all(np.isfinite(lp)) and np.all(np.isfinite(g)), (cid, team)
        assert_close_to_reference(lp, g, lp_mp, S, g_mp, G, (cid, team))
        assert_close_to_reference(lp, g, lo, S, go, G, (cid, team, "oracle"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_device_function_matches_the_oracle_on_the_builders(name):
    from oracle import ir_numpy_beta
    from pymc_b200 import engine

    m = BUILDERS[name]()
    cm = engine.CompiledModel(m)  # default path: no hand kernel takes it
    assert cm.spec.name == "ir" and (m.n > 256) == name.endswith("cta")
    f = ir_numpy_beta.make_logp(m)
    Q = m.initial_point() + np.random.default_rng(0).uniform(-1.0, 1.0, (9, m.n))
    lp, g = cm.logp_dlogp(Q)
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12
    assert np.max(np.abs(g - go) / np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))) <= 1e-12
    lp2, g2 = cm.logp_dlogp(Q)
    assert np.array_equal(lp, lp2) and np.array_equal(g, g2)


@pytest.mark.gpu
def test_device_pointwise_keeps_the_digits_of_small_counts():
    """The pointwise kernel on every BetaBinomial catalogue case: each observation with y <= 20 within 1e-12 (|log f_i| +
    1) of the reference, at a and b up to 1e8."""
    from pymc_b200 import engine

    checked = 0
    for cid in CASE_IDS:
        m = build(cid)
        if not any(L.dist == "beta_binomial_logit" for L in m.likelihoods):
            continue
        cm = engine.CompiledModel(m, specialise=False)
        for q in points(m, cid):
            checked += _small_counts_within(lambda k, L: cm.pointwise_loglik(q[None], lik=k)[0], cid, q)
    assert checked > 100


@pytest.mark.gpu
@pytest.mark.parametrize("name,eps", [("beta_var", 0.05), ("beta_binomial_var", 0.05), ("beta_binomial_var_cta", 0.01)])
def test_fixed_step_nuts_matches_the_oracle_sampler(name, eps):
    from oracle import ir_numpy_beta

    m = BUILDERS[name]()
    fixed_step_against_oracle(m, ir_numpy_beta.make_logp(m), eps)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle():
    from oracle import ir_numpy_beta

    m = ir.beta_regression_ir("beta_binomial", "var")
    fixed_step_against_oracle(m, ir_numpy_beta.make_logp(m), 0.2, dense_cov=random_dense_cov(m.n, 2, 0.02, 0.05, 12),
                              C=2, T=10)


@pytest.mark.gpu
def test_adaptive_beta_run_with_a_random_phi_matches_the_oracle_posterior():
    """64 device chains against 8 oracle chains (NUTS with diagonal mass adaptation) on the Beta regression with a random
    phi: posterior means within 5 SE, standard deviations within 25 %, divergences below 2 %."""
    from oracle import ir_numpy_beta

    m = ir.beta_regression_ir("beta", "var")
    adaptive_against_oracle(m, ir_numpy_beta.make_logp(m), chain_seed=23, spread=1, philox_seed=5, oracle_seed=200,
                            se_bound=5.0, max_divergence=0.02)


def _scipy_on_draws(m, q):
    from oracle import ir_numpy_beta

    f = ir_numpy_beta.make_logp(m)
    L = m.likelihoods[0]
    out = np.empty(q.shape[:-1] + (len(L.y),))
    for ix in np.ndindex(*q.shape[:-1]):
        x, _ = f.constrained(q[ix])
        out[ix] = scipy_pointwise(L, f.eta(L, x)[0], f.param(L, x)[0])
    return out


@pytest.mark.gpu
def test_pointwise_log_likelihood_and_the_log_likelihood_group_match_scipy():
    import pymc_b200
    from pymc_b200 import engine

    for dist, phi in SCIPY_BUILDS:
        m = ir.beta_regression_ir(dist, phi, n_obs=120)
        cm = engine.CompiledModel(m, specialise=False)
        q = m.initial_point() + np.random.default_rng(4).uniform(-0.5, 0.5, (2, 3, m.n))
        ll = cm.pointwise_loglik(q)
        assert ll.shape == (2, 3, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, _scipy_on_draws(m, q), rtol=1e-11, atol=1e-11, err_msg=f"{dist} {phi}")
    for m in (ir.beta_regression_ir("beta", "var"), ir.beta_regression_ir("beta_binomial", "var")):
        res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, keep_untransformed=True,
                                         idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
        ll = res.log_likelihood["y"]
        assert ll.shape == (4, 20, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, _scipy_on_draws(m, res.unconstrained), rtol=1e-11, atol=1e-11)
