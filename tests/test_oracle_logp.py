"""CPU: pins oracle/logp_numpy.py the way the reference pins its densities -- against scipy.stats
compositions (pymc/testing.py:311-418 check_logp), closed-form values from the reference's own tests,
and central finite differences for the hand-derived gradients."""
import numpy as np
import pytest
from b200_helpers import fd_grad
from scipy import stats as st

from oracle import logp_numpy as L
from pymc_b200 import models


def test_normal_matches_scipy():
    # tests/distributions/test_continuous.py:273-280
    x, mu, s = np.array([-2.1, 0.0, 0.3, 5.0]), 0.7, 1.9
    np.testing.assert_allclose(L.normal_logp(x, mu, s), st.norm.logpdf(x, mu, s), rtol=0, atol=1e-13)


def test_halfcauchy_log_matches_scipy():
    # tests/distributions/test_continuous.py:637-643 (HalfCauchy) + log transform Jacobian
    for z in (-3.0, 0.0, 1.7, 4.0):
        val, dz = L.halfcauchy_log_logp(z, 5.0)
        assert abs(val - (st.halfcauchy.logpdf(np.exp(z), scale=5.0) + z)) < 1e-13
        h = 1e-6
        assert abs(dz - (L.halfcauchy_log_logp(z + h, 5.0)[0] - L.halfcauchy_log_logp(z - h, 5.0)[0]) / (2 * h)) < 1e-8


def test_eight_schools_against_scipy_composition():
    spec = models.eight_schools()
    f = L.make_logp(spec)
    rng = np.random.default_rng(0)
    for _ in range(5):
        q = rng.normal(size=10)
        mu, ltau, tt = q[0], q[1], q[2:]
        tau = np.exp(ltau)
        want = (st.norm.logpdf(mu, 0, 5) + st.halfcauchy.logpdf(tau, scale=5) + ltau + st.norm.logpdf(tt).sum()
                + st.norm.logpdf(spec.data["y"], mu + tau * tt, spec.data["sigma"]).sum())
        assert abs(f(q)[0] - want) < 1e-11


def test_eight_schools_known_answer():
    # SURVEY 8c: produced by the verbatim reference code + this logp
    lp, g = L.make_logp(models.eight_schools())(np.zeros(10))
    assert lp == pytest.approx(-43.43563727714813, abs=1e-12)
    np.testing.assert_allclose(g[:3], [0.46353275, 0.92307692, 0.12444444], atol=1e-8)


def test_radon_against_scipy_composition():
    spec = models.radon()
    f = L.make_logp(spec)
    J = 85
    rng = np.random.default_rng(1)
    q = spec.initial_point() + rng.uniform(-1, 1, spec.n)
    mu_a, lsa, mu_b, lsb = q[:4]
    a, b, le = q[4 : 4 + J], q[4 + J : 4 + 2 * J], q[-1]
    idx, x, y = spec.data["county_idx"], spec.data["floor"], spec.data["y"]
    m = (mu_a + np.exp(lsa) * a)[idx] + (mu_b + np.exp(lsb) * b)[idx] * x
    want = (st.norm.logpdf(mu_a, 0, 100**2) + st.norm.logpdf(mu_b, 0, 100**2)
            + sum(st.halfcauchy.logpdf(np.exp(z), scale=5) + z for z in (lsa, lsb, le))
            + st.norm.logpdf(a).sum() + st.norm.logpdf(b).sum() + st.norm.logpdf(y, m, np.exp(le)).sum())
    assert abs(f(q)[0] - want) < 1e-9
    assert spec.n == 175 and len(y) == 919 and np.bincount(idx, minlength=J).min() >= 1


def test_logistic_against_scipy_composition():
    spec = models.logistic(n_rows=200, n_features=5, seed=3)
    f = L.make_logp(spec)
    q = np.random.default_rng(2).normal(size=5) * 0.5
    p = 1 / (1 + np.exp(-(spec.data["X"] @ q)))
    want = st.bernoulli.logpmf(spec.data["y"], p).sum() + st.norm.logpdf(q).sum()
    assert abs(f(q)[0] - want) < 1e-10


def test_stochvol_against_scipy_composition():
    # AR(1) logp == the equivalent Normal regression (tests/distributions/test_timeseries.py:467-504)
    spec = models.stochvol(T=50, seed=4)
    f = L.make_logp(spec)
    rng = np.random.default_rng(3)
    q = spec.initial_point() + rng.uniform(-0.5, 0.5, spec.n)
    mu, z, ls, h = q[0], q[1], q[2], q[3:]
    phi = 2 / (1 + np.exp(-z)) - 1
    sig = np.exp(ls)
    interval_jac = np.log(2.0) - 2 * np.log1p(np.exp(-z)) - z  # log(b-a) - 2 softplus(-z) - z
    want = (st.norm.logpdf(mu, 0, 5) + st.uniform.logpdf(phi, -1, 2) + interval_jac
            + st.expon.logpdf(sig, scale=0.1) + ls
            + st.norm.logpdf(h[0], 0, 1) + st.norm.logpdf(h[1:], phi * h[:-1], sig).sum()
            + st.norm.logpdf(spec.data["y"], 0, np.exp((mu + h) / 2)).sum())
    assert abs(f(q)[0] - want) < 1e-10


def test_mvgauss_against_scipy():
    spec = models.mvgauss(n=12, seed=5)
    f = L.make_logp(spec)
    q = np.random.default_rng(4).normal(size=12)
    want = st.multivariate_normal.logpdf(q, np.zeros(12), spec.data["cov"])
    assert abs(f(q)[0] - want) < 1e-10


@pytest.mark.parametrize("builder", [
    lambda: models.std_normal(7), models.eight_schools, lambda: models.radon(60, 9, 2),
    lambda: models.logistic(100, 6, 1), lambda: models.stochvol(30, 2), lambda: models.mvgauss(9, 3),
])
def test_gradients_by_central_differences(builder):
    spec = builder()
    f = L.make_logp(spec)
    rng = np.random.default_rng(5)
    q = spec.initial_point() + rng.uniform(-0.7, 0.7, spec.n)
    g = f(q)[1]
    np.testing.assert_allclose(g, fd_grad(f, q), rtol=2e-6, atol=2e-6)


def test_model_dlogp_closed_form():
    """tests/model/test_core.py:1081-1129 style: Normal value var -> d/dx logp = -(x-mu)/sigma^2."""
    f = L.make_logp(models.std_normal(3))
    lp, g = f(np.array([0.0, 1.0, -2.0]))
    np.testing.assert_allclose(g, [0.0, -1.0, 2.0])
    assert lp == pytest.approx(st.norm.logpdf([0.0, 1.0, -2.0]).sum())


def test_compiled_radon_logp_equals_the_numpy_form():
    """oracle/c/radon_logp.c (the compiled-code logp of bench.py's CPU baseline) against RadonLogp, logp and gradient."""
    import os
    import shutil
    import subprocess

    from oracle import logp_numpy
    from pymc_b200 import models

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.isfile(logp_numpy.RadonLogpC.LIB):
        if shutil.which("gcc") is None or shutil.which("make") is None:
            pytest.skip("no C toolchain to build oracle/c")
        subprocess.check_call(["make", "-C", os.path.join(root, "oracle", "c")])
    spec = models.radon()
    f, fc = logp_numpy.make_logp(spec), logp_numpy.make_logp(spec, compiled=True)
    assert type(fc).__name__ == "RadonLogpC"
    rng = np.random.default_rng(3)
    for _ in range(20):
        q = spec.initial_point() + rng.uniform(-2, 2, spec.n)
        a, ga = f(q)
        b, gb = fc(q)
        assert abs(a - b) <= 1e-12 * abs(a) and np.max(np.abs(ga - gb)) <= 1e-12 * np.max(np.abs(ga))
    # models without a C build fall back to the NumPy form
    assert type(logp_numpy.make_logp(models.eight_schools(), compiled=True)).__name__ == "EightSchoolsLogp"
