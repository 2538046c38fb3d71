"""TEST INFRASTRUCTURE ONLY -- NumPy/SciPy restatement of the compiled ``logp/dlogp`` callable.

The reference builds ``q[n] -> (logp, dlogp[n])`` with PyTensor (model/core.py:232-267); PyTensor
(pinned ``>=3.2.2,<3.3``, requirements.txt:6) is absent from /root/reference and from this image, so
this file restates the *published formulas* the PyTensor graph encodes.  Each density cites the
reference line it follows; gradients are hand-derived (SURVEY.md Appendix C) and pinned by
``tests/test_oracle_logp.py`` against ``scipy.stats`` compositions (what the reference's own
``check_logp`` tests do, pymc/testing.py:311-418), central finite differences, and the reference
test-suite's closed-form values.

Conventions copied from the reference:
  * q is the concatenation of transformed value variables in registration order
    (pytensorf.py:575-595);
  * a log-transformed RV contributes its Jacobian ``+z`` (logprob/transforms.py:880-891);
    the interval transform contributes ``log(b-a) - 2 softplus(-z) - z`` (:1060-1062);
  * factors are summed with no reweighting (model/core.py:688-690);
  * stable forms: ``log sigmoid(x) = -softplus(-x)`` as PyTensor's ``stabilize`` rewrite produces
    (applied at pytensorf.py:1089-1093).

Only tests/, bench.py's cpu_baseline leg and __graft_entry__.smoke() may import this module.
"""
from __future__ import annotations

import os

import numpy as np

LOG_2PI = np.log(2.0 * np.pi)
HALF_LOG_2PI = 0.5 * LOG_2PI


def softplus(x):
    x = np.asarray(x, dtype=np.float64)
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def sigmoid(x):
    x = np.asarray(x, dtype=np.float64)
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def normal_logp(x, mu, sigma):
    """Normal.logp, distributions/continuous.py:526-527."""
    z = (x - mu) / sigma
    return -0.5 * z * z - HALF_LOG_2PI - np.log(sigma)


def halfcauchy_log_logp(z, beta):
    """HalfCauchy(beta) on x=exp(z) plus the log-transform Jacobian.

    Cauchy.logp continuous.py:2287-2288, HalfCauchy.logp :2383-2385, LogTransform jacobian
    logprob/transforms.py:880-891.  Returns (value, d/dz)."""
    x = np.exp(z)
    u = (x / beta) ** 2
    val = np.log(2.0) - np.log(np.pi) - np.log(beta) - np.log1p(u) + z
    return val, 1.0 - 2.0 * u / (1.0 + u)


class StdNormalLogp:
    def __init__(self, spec):
        self.n = spec.n

    def __call__(self, q):
        return float(-0.5 * np.dot(q, q) - self.n * HALF_LOG_2PI), -q


class EightSchoolsLogp:
    """SURVEY Appendix C-1.  q = [mu, log tau, theta_t[8]]."""

    def __init__(self, spec):
        self.y = spec.data["y"]
        self.s = spec.data["sigma"]
        self.n = spec.n

    def __call__(self, q):
        mu, ltau, tt = q[0], q[1], q[2:]
        tau = np.exp(ltau)
        theta = mu + tau * tt
        hc, dhc = halfcauchy_log_logp(ltau, 5.0)
        logp = (
            normal_logp(mu, 0.0, 5.0)
            + hc
            + np.sum(normal_logp(tt, 0.0, 1.0))
            + np.sum(normal_logp(self.y, theta, self.s))
        )
        r = (self.y - theta) / self.s**2
        g = np.empty(self.n)
        g[0] = -mu / 25.0 + np.sum(r)
        g[1] = dhc + tau * np.sum(r * tt)
        g[2:] = -tt + tau * r
        return float(logp), g


class RadonLogp:
    """SURVEY Appendix C-2; model benchmarks/benchmarks/benchmarks.py:34-45 (note sigma=100**2)."""

    def __init__(self, spec):
        self.idx = spec.data["county_idx"].astype(np.int64)
        self.x = spec.data["floor"]
        self.y = spec.data["y"]
        self.J = spec.meta["n_counties"]
        self.n = spec.n

    def __call__(self, q):
        J = self.J
        mu_a, lsa, mu_b, lsb = q[0], q[1], q[2], q[3]
        a, b, leps = q[4 : 4 + J], q[4 + J : 4 + 2 * J], q[4 + 2 * J]
        sa, sb, eps = np.exp(lsa), np.exp(lsb), np.exp(leps)
        alpha = mu_a + sa * a
        beta = mu_b + sb * b
        m = alpha[self.idx] + beta[self.idx] * self.x
        d = self.y - m
        hca, dhca = halfcauchy_log_logp(lsa, 5.0)
        hcb, dhcb = halfcauchy_log_logp(lsb, 5.0)
        hce, dhce = halfcauchy_log_logp(leps, 5.0)
        S = 100.0**2
        logp = (
            normal_logp(mu_a, 0.0, S)
            + normal_logp(mu_b, 0.0, S)
            + hca
            + hcb
            + hce
            + np.sum(normal_logp(a, 0.0, 1.0))
            + np.sum(normal_logp(b, 0.0, 1.0))
            + np.sum(normal_logp(self.y, m, eps))
        )
        r = d / eps**2
        Ga = np.bincount(self.idx, weights=r, minlength=J)
        Gb = np.bincount(self.idx, weights=r * self.x, minlength=J)
        g = np.empty(self.n)
        g[0] = -mu_a / S**2 + Ga.sum()
        g[1] = dhca + sa * np.dot(a, Ga)
        g[2] = -mu_b / S**2 + Gb.sum()
        g[3] = dhcb + sb * np.dot(b, Gb)
        g[4 : 4 + J] = -a + sa * Ga
        g[4 + J : 4 + 2 * J] = -b + sb * Gb
        g[4 + 2 * J] = dhce + np.sum(d * d) / eps**2 - len(self.y)
        return float(logp), g


class LogisticLogp:
    """SURVEY Appendix C-3; Bernoulli(logit_p) discrete.py:351-367 with the stabilised
    ``log sigmoid`` forms: y*eta - softplus(eta)."""

    def __init__(self, spec):
        self.X = spec.data["X"]
        self.y = spec.data["y"].astype(np.float64)
        self.n = spec.n

    def __call__(self, q):
        eta = self.X @ q
        logp = np.sum(self.y * eta - softplus(eta)) + np.sum(normal_logp(q, 0.0, 1.0))
        g = self.X.T @ (self.y - sigmoid(eta)) - q
        return float(logp), g


class StochVolLogp:
    """SURVEY Appendix C-4.  q = [mu, z_phi, log sigma, h[T]].

    AR(1) logp timeseries.py:646-676 (init Normal(0,1) on h0, innovations Normal(0,sigma));
    Uniform(-1,1)+interval continuous.py:309, transforms.py:1026-1073; Exponential(lam=10)
    continuous.py:1478-1480 with mu=1/lam."""

    def __init__(self, spec):
        self.y = spec.data["y"]
        self.T = spec.meta["T"]
        self.n = spec.n

    def __call__(self, q):
        T = self.T
        mu, zphi, lsig = q[0], q[1], q[2]
        h = q[3:]
        s = sigmoid(zphi)
        phi = 2.0 * s - 1.0
        sig = np.exp(lsig)
        e = h[1:] - phi * h[:-1]
        w = self.y**2 * np.exp(-(mu + h))
        logp = (
            normal_logp(mu, 0.0, 5.0)
            + (-2.0 * softplus(-zphi) - zphi)
            + (np.log(10.0) - 10.0 * sig + lsig)
            + normal_logp(h[0], 0.0, 1.0)
            + np.sum(normal_logp(e, 0.0, sig))
            + np.sum(-0.5 * w - HALF_LOG_2PI - 0.5 * (mu + h))
        )
        g = np.empty(self.n)
        dh = 0.5 * w - 0.5
        es = e / sig**2
        gh = dh.copy()
        gh[1:] -= es
        gh[:-1] += phi * es
        gh[0] -= h[0]
        g[0] = -mu / 25.0 + np.sum(dh)
        ez = np.exp(-abs(zphi))  # s (1 - s) = e / (1 + e)^2: no cancellation in 1 - s at large |zphi|
        g[1] = (1.0 - 2.0 * s) + 2.0 * (ez / ((1.0 + ez) * (1.0 + ez))) * np.sum(es * h[:-1])
        g[2] = 1.0 - 10.0 * sig + np.sum(e * e) / sig**2 - (T - 1)
        g[3:] = gh
        return float(logp), g


class MvGaussLogp:
    """SURVEY Appendix C-5; MvNormal.logp multivariate.py:275-295 via the Cholesky factor
    (quaddist_chol :165-185): -n/2 log 2pi - sum log L_ii - 1/2 |L^-1 x|^2.  Gradient -P x."""

    def __init__(self, spec):
        import scipy.linalg as sl

        self._sl = sl
        self.L = spec.data["L"]
        self.P = spec.data["prec"]
        self.logdet = spec.meta["logdet_L"]
        self.n = spec.n

    def __call__(self, q):
        w = self._sl.solve_triangular(self.L, q, lower=True)
        logp = -0.5 * self.n * LOG_2PI - self.logdet - 0.5 * np.dot(w, w)
        return float(logp), -(self.P @ q)


_BY_KIND = {
    0: StdNormalLogp,
    1: EightSchoolsLogp,
    2: RadonLogp,
    3: LogisticLogp,
    4: StochVolLogp,
    5: MvGaussLogp,
}


class RadonLogpC:
    """The same function as ``RadonLogp`` from oracle/c/radon_logp.c (gcc -O3, built by ``make -C oracle/c`` /
    ``__graft_entry__.build()``): what bench.py's CPU baseline calls, so that a logp/dlogp evaluation costs what compiled code
    costs -- the reference runs this function as a PyTensor C thunk (model/core.py:232-267)."""

    LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "libradon_logp.so")

    def __init__(self, spec):
        import ctypes as C

        lib = C.CDLL(self.LIB)
        fn = lib.radon_logp_dlogp
        fn.restype = C.c_double
        fn.argtypes = [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        self._fn = fn
        self.idx = np.ascontiguousarray(spec.data["county_idx"], dtype=np.int64)
        self.x = np.ascontiguousarray(spec.data["floor"], dtype=np.float64)
        self.y = np.ascontiguousarray(spec.data["y"], dtype=np.float64)
        self.J, self.n, self.N = int(spec.meta["n_counties"]), spec.n, len(self.y)
        self._Ga, self._Gb = np.empty(self.J), np.empty(self.J)
        self._args = (self.J, self.N, self.idx.ctypes.data, self.x.ctypes.data, self.y.ctypes.data)
        self._scr = (self._Ga.ctypes.data, self._Gb.ctypes.data)

    def __call__(self, q):
        q = np.ascontiguousarray(q, dtype=np.float64)
        g = np.empty(self.n)
        lp = self._fn(q.ctypes.data, *self._args, g.ctypes.data, *self._scr)
        return float(lp), g


def compiled_logp_available(spec) -> bool:
    return spec.name == "radon" and os.path.isfile(RadonLogpC.LIB)


def make_logp(spec, compiled: bool = False):
    """ModelSpec -> callable q -> (logp, grad).  ``compiled=True``: the plain-C build where one exists (Radon), for the CPU
    baseline; parity tests and goldens use the NumPy forms."""
    if compiled and compiled_logp_available(spec):
        return RadonLogpC(spec)
    return _BY_KIND[spec.kind](spec)
