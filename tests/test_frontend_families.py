"""from_pymc on real PyMC models with Binomial, NegativeBinomial and Gamma likelihoods: the lowering is checked against the
model's own compiled logp/dlogp (pymc/model/core.py:464-529).  Skipped where PyMC is not installed."""
import numpy as np
import pytest

pm = pytest.importorskip("pymc")


def _check(model, rtol=1e-9):
    from oracle import ir_numpy_families
    from pymc_b200 import from_pymc

    m = from_pymc(model)
    f = model.logp_dlogp_function(ravel_inputs=True)
    f.set_extra_values({})
    g = ir_numpy_families.make_logp(m)
    rng = np.random.default_rng(0)
    for _ in range(3):
        q = m.initial_point() + rng.uniform(-0.5, 0.5, m.n)
        lp_ref, dlp_ref = f(q)
        lp, dlp = g(q)
        np.testing.assert_allclose(lp, lp_ref, rtol=rtol)
        np.testing.assert_allclose(dlp, dlp_ref, rtol=1e-7, atol=1e-9)
    return m


@pytest.mark.parametrize("spelling", ["logit_p", "invlogit"])
def test_binomial_lowers(spelling):
    rng = np.random.default_rng(1)
    N, G = 60, 6
    g = rng.integers(0, G, N)
    n = rng.integers(1, 30, N)
    y = rng.binomial(n, 0.3)
    with pm.Model() as model:
        mu = pm.Normal("mu", 0, 2)
        s = pm.HalfNormal("s", 1)
        a = pm.Normal("a", mu, s, shape=G)
        eta = a[g]
        if spelling == "logit_p":
            pm.Binomial("y", n=n, logit_p=eta, observed=y)
        else:
            pm.Binomial("y", n=n, p=pm.math.invlogit(eta), observed=y)
    assert _check(model).likelihoods[0].dist == "binomial_logit"


@pytest.mark.parametrize("random_alpha", [True, False])
def test_negative_binomial_lowers(random_alpha):
    rng = np.random.default_rng(2)
    N = 80
    x = rng.standard_normal(N)
    y = rng.negative_binomial(2.0, 0.4, N)
    with pm.Model() as model:
        b0 = pm.Normal("b0", 0, 2)
        b1 = pm.Normal("b1", 0, 1)
        alpha = pm.Exponential("alpha", 1.0) if random_alpha else 2.5
        pm.NegativeBinomial("y", mu=pm.math.exp(b0 + b1 * x), alpha=alpha, observed=y)
    assert _check(model).likelihoods[0].dist == "negative_binomial_log"


@pytest.mark.parametrize("form", ["divide", "multiply"])
def test_gamma_lowers(form):
    rng = np.random.default_rng(3)
    N = 70
    x = rng.standard_normal(N)
    y = rng.gamma(3.0, 0.7, N)
    with pm.Model() as model:
        b0 = pm.Normal("b0", 0, 2)
        b1 = pm.Normal("b1", 0, 1)
        a = pm.HalfNormal("alpha", 2.0)
        eta = b0 + b1 * x
        beta = a / pm.math.exp(eta) if form == "divide" else a * pm.math.exp(-eta)
        pm.Gamma("y", alpha=a, beta=beta, observed=y)
    assert _check(model).likelihoods[0].dist == "gamma_log"


def test_other_spellings_are_refused():
    from pymc_b200 import from_pymc

    with pm.Model() as model:
        b0 = pm.Normal("b0", 0, 1)
        pm.Gamma("y", mu=pm.math.exp(b0), sigma=1.0, observed=np.array([1.0, 2.0]))
    with pytest.raises(NotImplementedError):
        from_pymc(model)
