"""CPU: ``from_pymc`` on imitation graphs (tests/test_frontend_mock.py's stand-ins) of Beta regression observations:
pm.Beta(mu=invlogit(eta), nu=phi) and pm.Beta(alpha=mu * phi, beta=(1 - mu) * phi), which both build a BetaRV with dist
params (mu * phi, (1 - mu) * phi), and pm.BetaBinomial(alpha=mu * phi, beta=(1 - mu) * phi, n=trials), a BetaBinomialRV
with dist params (n, alpha, beta).  Each accepted spelling must lower to an IR whose oracle density equals scipy.stats';
the other forms are refused by name.  A real PyMC model goes through the same matcher under importorskip("pymc")."""
import re

import numpy as np
import pytest
from scipy import stats
from test_frontend_mock import Constant, FakeModel, LogTransform, bcast, elem, fake_pytensor, rv  # noqa: F401

from oracle.ir_numpy_beta import make_logp
from pymc_b200 import ir

N = 24


def _model(rng, obs, phi="free"):
    """b0 + b1 x as a graph, phi ~ Gamma(2, 0.1) (or a constant), sigma ~ HalfNormal(1); obs(M, eta, phi, sigma) adds the
    observed RV."""
    x = rng.standard_normal(N)
    M = FakeModel("beta")
    b0 = M.free(rv("NormalRV", "b0", Constant(0.0), Constant(1.5)), 1)
    b1 = M.free(rv("NormalRV", "b1", Constant(0.0), Constant(1.0)), 1)
    p = M.free(rv("GammaRV", "phi", Constant(2.0), Constant(10.0)), 1, LogTransform()) if phi == "free" else Constant(phi)
    s = M.free(rv("HalfNormalRV", "sigma", Constant(0.0), Constant(1.0)), 1, LogTransform())
    eta = elem("Add", bcast(b0), elem("Mul", bcast(b1), Constant(x)))
    obs(M, eta, p, s)
    return M, x


def _ab(eta, p, order="mu_first", mean="Sigmoid"):
    """alpha = mu * phi and beta = (1 - mu) * phi, as get_alpha_beta and a hand-written alpha / beta both build them."""
    mu = elem(mean, eta)
    ph = bcast(p) if not isinstance(p, Constant) else p
    one_minus = elem("Sub", Constant(1.0), mu)
    if order == "mu_first":
        return elem("Mul", mu, ph), elem("Mul", one_minus, ph)
    return elem("Mul", ph, mu), elem("Mul", ph, one_minus)


SPELLINGS = [("beta", "mu_first"), ("beta", "phi_first"), ("beta_binomial", "mu_first"), ("beta_binomial", "phi_first")]


@pytest.mark.parametrize("phi", ["free", 7.5])
@pytest.mark.parametrize("dist,order", SPELLINGS)
def test_beta_graphs_lower_to_the_beta_likelihoods(fake_pytensor, dist, order, phi):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(21)
    trials = rng.integers(0, 30, N).astype(np.float64)
    p = rng.beta(2.0, 3.0, N)
    y = p if dist == "beta" else rng.binomial(trials.astype(np.int64), p).astype(np.float64)

    def obs(M, eta, ph, s):
        a, b = _ab(eta, ph, order)
        M.observe(rv("BetaRV", "y", a, b) if dist == "beta" else rv("BetaBinomialRV", "y", Constant(trials), a, b), y)

    M, x = _model(rng, obs, phi)
    m = from_pymc(M)
    L = m.likelihoods[0]
    assert L.dist == ("beta_logit" if dist == "beta" else "beta_binomial_logit")
    assert L.phi == (ir.Ref("phi_log__") if phi == "free" else 7.5) and L.sigma is None and L.alpha is None
    assert (L.trials is None) if dist == "beta" else np.array_equal(L.trials, trials)
    f = make_logp(m)
    q = m.initial_point() + rng.uniform(-0.5, 0.5, m.n)
    xs, _ = f.constrained(q)
    P = m.constrain(q)
    mu = 1.0 / (1.0 + np.exp(-(P["b0"] + P["b1"] * x)))
    ph = P["phi"] if phi == "free" else phi
    want = stats.beta.logpdf(y, mu * ph, (1 - mu) * ph) if dist == "beta" else \
        stats.betabinom.logpmf(y, trials, mu * ph, (1 - mu) * ph)
    np.testing.assert_allclose(f.loglik(L, xs), want, rtol=1e-10, atol=1e-10)


def test_constant_trials_are_kept(fake_pytensor):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(22)
    y = rng.binomial(12, 0.4, N).astype(np.float64)
    M, _ = _model(rng, lambda M, eta, p, s: M.observe(rv("BetaBinomialRV", "y", Constant(12.0), *_ab(eta, p)), y))
    L = from_pymc(M).likelihoods[0]
    assert L.dist == "beta_binomial_logit" and L.trials == 12.0


def test_other_forms_are_refused_by_name(fake_pytensor):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(23)
    y = rng.beta(2.0, 2.0, N)
    yc = rng.binomial(10, 0.5, N).astype(np.float64)

    def model(obs):
        return _model(rng, obs)[0]

    def obs_with(r, data=y):
        return lambda M, eta, p, s: M.observe(r(M, eta, p, s), data)

    def kappa(eta, s):  # Beta(mu, sigma): kappa = mu (1 - mu) / sigma**2 - 1, alpha = mu kappa, beta = (1 - mu) kappa
        mu = elem("Sigmoid", eta)
        k = elem("Sub", elem("TrueDiv", elem("Mul", mu, elem("Sub", Constant(1.0), mu)), elem("Pow", bcast(s), Constant(2.0))),
                 Constant(1.0))
        return elem("Mul", mu, k), elem("Mul", elem("Sub", Constant(1.0), mu), k)

    per_obs = Constant(np.linspace(2.0, 9.0, N))
    cases = [
        ("the kappa form", obs_with(lambda M, eta, p, s: rv("BetaRV", "y", *kappa(eta, s)))),
        ("constant alpha and beta with no predictor", obs_with(lambda M, eta, p, s: rv("BetaRV", "y", Constant(2.0), Constant(3.0)))),
        ("per-observation or vector phi",
         obs_with(lambda M, eta, p, s: rv("BetaRV", "y", elem("Mul", elem("Sigmoid", eta), per_obs),
                                          elem("Mul", elem("Sub", Constant(1.0), elem("Sigmoid", eta)), per_obs)))),
        ("phi that is an expression",
         obs_with(lambda M, eta, p, s: rv("BetaRV", "y", *_ab(eta, elem("Mul", bcast(p), bcast(s)))))),
        ("a mean other than invlogit", obs_with(lambda M, eta, p, s: rv("BetaRV", "y", *_ab(eta, p, mean="Exp")))),
        ("random trials", obs_with(lambda M, eta, p, s: rv("BetaBinomialRV", "y", bcast(p), *_ab(eta, p)), yc)),
        ("beta must be (1 - mu) * phi",
         obs_with(lambda M, eta, p, s: rv("BetaRV", "y", _ab(eta, p)[0], elem("Mul", elem("Sub", Constant(1.0), elem("Sigmoid", eta)),
                                                                                  bcast(s))))),
        ("write the likelihood as pm.BetaBinomial",
         obs_with(lambda M, eta, p, s: rv("BetaBinomialRV", "y", Constant(10.0), elem("Sigmoid", eta), bcast(p)), yc)),
    ]
    for what, obs in cases:
        with pytest.raises(NotImplementedError, match=re.escape(what)):
            from_pymc(model(obs))


def test_a_real_pymc_beta_regression_lowers():
    pm = pytest.importorskip("pymc")
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(24)
    x = rng.standard_normal(40)
    y = rng.beta(3.0, 4.0, 40)
    n = rng.integers(1, 20, 40)
    with pm.Model() as model:
        b0 = pm.Normal("b0", 0.0, 1.5)
        b1 = pm.Normal("b1", 0.0, 1.0)
        phi = pm.Gamma("phi", 2.0, 0.1)
        mu = pm.math.invlogit(b0 + b1 * x)
        pm.Beta("y", mu=mu, nu=phi, observed=y)
        pm.BetaBinomial("c", alpha=mu * phi, beta=(1 - mu) * phi, n=n, observed=rng.binomial(n, 0.4))
    m = from_pymc(model)
    assert [L.dist for L in m.likelihoods] == ["beta_logit", "beta_binomial_logit"]
    f = make_logp(m)
    q = m.initial_point() + rng.uniform(-0.3, 0.3, m.n)
    lp = f(q)[0]
    want = model.compile_logp()(dict(zip([v.name for v in model.value_vars], _split(m, q, model))))
    assert abs(lp - want) <= 1e-9 * abs(want)


def _split(m, q, model):
    off = m.offsets()
    return [q[off[v.name]: off[v.name] + m.var(v.name).size].reshape(model.initial_point()[v.name].shape)
            for v in model.value_vars]
