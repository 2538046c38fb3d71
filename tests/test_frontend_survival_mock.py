"""CPU: ``from_pymc`` on imitation graphs (tests/test_frontend_mock.py's stand-ins) of survival observations:
pm.Weibull(alpha, beta=exp(eta)) (a WeibullBetaRV with dist params (alpha, beta)), pm.Exponential(scale=exp(eta)) and
pm.Exponential(lam=exp(-eta)) (an ExponentialRV whose one parameter is the scale, reciprocal(lam)), pm.LogNormal(eta,
sigma), each plain, under pm.Censored (a CensoredRV of the base) and under pm.Truncated (a TruncatedRV: the base RV's
inputs, then lower and upper).  Each graph must lower to the expected IR, whose oracle density equals a scipy.stats
composition; the other forms are refused by name."""
import numpy as np
import pytest
from scipy import stats
from test_frontend_bounded_mock import truncated_rv
from test_frontend_mock import Constant, FakeModel, LogTransform, bcast, elem, fake_pytensor, rv  # noqa: F401

from oracle.ir_numpy_survival import make_logp
from pymc_b200 import ir

N = 24


def _model(rng, obs, alpha="free"):
    """b0 + b1 x as a graph, alpha ~ HalfNormal(2) (or a constant) and sigma ~ HalfNormal(1); obs(M, eta, alpha, sigma)
    adds the observed RV."""
    x = rng.standard_normal(N)
    M = FakeModel("survival")
    b0 = M.free(rv("NormalRV", "b0", Constant(0.0), Constant(2.0)), 1)
    b1 = M.free(rv("NormalRV", "b1", Constant(0.0), Constant(1.0)), 1)
    a = M.free(rv("HalfNormalRV", "alpha", Constant(0.0), Constant(2.0)), 1, LogTransform()) if alpha == "free" else \
        Constant(alpha)
    s = M.free(rv("HalfNormalRV", "sigma", Constant(0.0), Constant(1.0)), 1, LogTransform())
    eta = elem("Add", bcast(b0), elem("Mul", bcast(b1), Constant(x)))
    obs(M, eta, a, s)
    return M, x


def _base(spelling, eta, a, s):
    if spelling == "weibull":
        return rv("WeibullBetaRV", None, bcast(a) if not isinstance(a, Constant) else a, elem("Exp", eta))
    if spelling == "exponential_scale":
        return rv("ExponentialRV", None, elem("Exp", eta))
    if spelling == "exponential_lam":
        return rv("ExponentialRV", None, elem("Reciprocal", elem("Exp", elem("Neg", eta))))
    return rv("LogNormalRV", None, eta, bcast(s))


SPELLINGS = ["weibull", "exponential_scale", "exponential_lam", "lognormal"]
FORMS = ["plain", "censored", "truncated"]


def _scipy(spelling, y, eta, a, s, form, lo, hi):
    d = stats.lognorm(s, scale=np.exp(eta)) if spelling == "lognormal" else \
        stats.weibull_min(a if spelling == "weibull" else 1.0, scale=np.exp(eta))
    if form == "censored":
        return np.where(y == hi, d.logsf(y), np.where(y == lo, d.logcdf(y), d.logpdf(y)))
    if form == "truncated":
        return d.logpdf(y) - np.log(d.sf(lo) - d.sf(hi))
    return d.logpdf(y)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("spelling", SPELLINGS)
def test_survival_graphs_lower_to_the_survival_likelihoods(fake_pytensor, spelling, form):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(11)
    y = rng.weibull(1.3, N) * 1.5
    lo, hi = 0.0, np.inf
    if form == "censored":  # right-censored at per-observation follow-up times, left-censored at one detection limit
        lo = float(np.quantile(y, 0.15))
        hi = np.where(rng.random(N) < 0.4, np.maximum(y * rng.uniform(0.5, 1.0, N), 2.0 * lo), np.inf)
        y = np.clip(y, lo, hi)
    elif form == "truncated":  # delayed entry
        lo = np.where(rng.random(N) < 0.3, 0.0, y * rng.uniform(0.2, 0.9, N))

    def obs(M, eta, a, s):
        base = _base(spelling, eta, a, s)
        if form == "plain":
            base.name = "y"
            M.observe(base, y)
        elif form == "censored":
            M.observe(rv("CensoredRV", "y", base, Constant(lo), Constant(hi)), y)
        else:
            params = base.owner.inputs[2:]
            op = {"weibull": "WeibullBetaRV", "lognormal": "LogNormalRV"}.get(spelling, "ExponentialRV")
            M.observe(truncated_rv("y", op, *params, lower=Constant(lo), upper=Constant(np.inf)), y)

    M, x = _model(rng, obs)
    m = from_pymc(M)
    L = m.likelihoods[0]
    fam = "lognormal" if spelling == "lognormal" else "weibull_log"
    assert L.dist == (fam if form == "plain" else f"{form}_{fam}")
    if spelling == "lognormal":
        assert L.sigma == ir.Ref("sigma_log__") and L.alpha is None
    else:
        assert L.alpha == (ir.Ref("alpha_log__") if spelling == "weibull" else 1.0) and L.sigma is None
    if form == "censored":
        assert L.lower == lo and np.array_equal(L.upper, hi)
    elif form == "truncated":
        assert np.array_equal(L.lower, lo) and L.upper is None
    f = make_logp(m)
    q = m.initial_point() + rng.uniform(-0.5, 0.5, m.n)
    xs, _ = f.constrained(q)
    P = m.constrain(q)
    eta = P["b0"] + P["b1"] * x
    want = _scipy(spelling, y, eta, P["alpha"], P["sigma"], form, np.broadcast_to(lo, (N,)), np.broadcast_to(hi, (N,)))
    np.testing.assert_allclose(f.loglik(L, xs), want, rtol=1e-10, atol=1e-10)


def test_a_constant_alpha_is_kept(fake_pytensor):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(12)
    y = rng.weibull(2.0, N)
    M, _ = _model(rng, lambda M, eta, a, s: M.observe(rv("WeibullBetaRV", "y", Constant(2.5), elem("Exp", eta)), y),
                  alpha=2.5)
    L = from_pymc(M).likelihoods[0]
    assert L.dist == "weibull_log" and L.alpha == 2.5


def test_other_forms_are_refused_by_name(fake_pytensor):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(13)
    y = rng.weibull(1.5, N) + 0.1

    def model(obs):
        return _model(rng, obs)[0]

    def obs_with(r):
        return lambda M, eta, a, s: M.observe(r(M, eta, a, s), y)

    cases = [
        ("write the likelihood as pm.Weibull", obs_with(lambda M, eta, a, s: rv("WeibullBetaRV", "y", bcast(a), eta))),
        ("per-observation or vector Weibull alpha",
         obs_with(lambda M, eta, a, s: rv("WeibullBetaRV", "y", Constant(np.linspace(1.0, 2.0, N)), elem("Exp", eta)))),
        ("Weibull alpha that is an expression",
         obs_with(lambda M, eta, a, s: rv("WeibullBetaRV", "y", elem("Mul", bcast(a), bcast(s)), elem("Exp", eta)))),
        ("write the likelihood as pm.Exponential",  # lam = exp(eta)
         obs_with(lambda M, eta, a, s: rv("ExponentialRV", "y", elem("Reciprocal", elem("Exp", eta))))),
        ("write the likelihood as pm.Exponential", obs_with(lambda M, eta, a, s: rv("ExponentialRV", "y", eta))),
        ("random bounds", obs_with(lambda M, eta, a, s: rv("CensoredRV", "y", rv("WeibullBetaRV", None, bcast(a), elem("Exp", eta)),
                                                           Constant(0.0), bcast(s)))),
        ("random bounds", obs_with(lambda M, eta, a, s: truncated_rv("y", "LogNormalRV", eta, bcast(s), lower=bcast(a),
                                                                     upper=Constant(np.inf)))),
        ("pm.Censored of a pm.Truncated", obs_with(lambda M, eta, a, s: rv(
            "CensoredRV", "y", truncated_rv(None, "WeibullBetaRV", bcast(a), elem("Exp", eta), lower=Constant(0.05),
                                            upper=Constant(np.inf)), Constant(0.0), Constant(3.0)))),
        ("pm.Censored of GammaRV", obs_with(lambda M, eta, a, s: rv("CensoredRV", "y", rv("GammaRV", None, bcast(a), elem("Exp", eta)),
                                                                    Constant(0.0), Constant(3.0)))),
        ("pm.Truncated of GammaRV", obs_with(lambda M, eta, a, s: truncated_rv("y", "GammaRV", bcast(a), elem("Exp", eta),
                                                                               lower=Constant(0.05), upper=Constant(np.inf)))),
    ]
    for what, obs in cases:
        with pytest.raises(NotImplementedError, match=what):
            from_pymc(model(obs))
