"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` with Beta regression
likelihoods (``BETA_LIKS``): ``beta_logit`` and ``beta_binomial_logit``.

Layered like oracle/ir_numpy_mixture.py: the rest of the model (every other factor, the prior of phi and every
transform) is evaluated by the oracle it is given (by default ir_numpy_mixture.make_logp, which covers every other factor
of the closed set).  This module adds the Beta factors with every constant, at mu = sigmoid(eta), a = phi mu and
b = phi (1 - mu), a and b both formed from one e = exp(-|eta|):

  beta_logit           Beta(mu, nu = phi), continuous.py:1131-1262 (alpha = mu nu, beta = (1 - mu) nu, :1238-1240):
                       log f = lgamma(phi) - lgamma(a) - lgamma(b) + (a - 1) log y + (b - 1) log1p(-y)
  beta_binomial_logit  BetaBinomial(n, a, b), discrete.py:178-262:
                       log f = binomln(n, y) + [lgamma(y + a) - lgamma(a)] + [lgamma(n - y + b) - lgamma(b)]
                               - [lgamma(n + phi) - lgamma(phi)]
                       each bracket lgamma(c + m) - lgamma(c) summed as sum_{j<m} log(c + j) below m = SUM_MAX, so a
                       small count keeps its digits however large c is

Pinned by tests/test_ir_beta.py against a 40-digit mpmath reference (itself checked against scipy.stats) and central
differences.  Only tests/ may import it.
"""
from __future__ import annotations

import dataclasses

import numpy as np
from scipy.special import digamma, gammaln

from oracle import ir_numpy_bounded, ir_numpy_mixture, ir_numpy_ordinal, ir_numpy_zero_inflated
from pymc_b200.ir import BETA_LIKS, ModelIR, Ref

SUM_MAX = 32  # the device's kIrBetaSumMax (csrc/ir_model.cuh)


def logit_parts(eta):
    """(mu, 1 - mu, mu (1 - mu)) from one e = exp(-|eta|)."""
    eta = np.asarray(eta, dtype=np.float64)
    e = np.exp(-np.abs(eta))
    h = 1.0 / (1.0 + e)
    return np.where(eta >= 0, h, e * h), np.where(eta >= 0, e * h, h), e * h * h


def rising(c, m):
    """(lgamma(c + m) - lgamma(c), digamma(c + m) - digamma(c)) of each element: sum_{j<m} log(c + j) and 1 / (c + j)
    below SUM_MAX, the lgamma / digamma differences from it on."""
    c, m = np.broadcast_arrays(np.asarray(c, dtype=np.float64), np.asarray(m, dtype=np.float64))
    small = m < SUM_MAX
    l, d = np.zeros(c.shape), np.zeros(c.shape)
    for j in range(SUM_MAX - 1):
        on = small & (j < m)
        t = np.where(on, c + j, 1.0)
        l += np.where(on, np.log(t), 0.0)
        d += np.where(on, 1.0 / t, 0.0)
    cb, mb = np.where(small, 1.0, c), np.where(small, 0.0, m)
    l = np.where(small, l, gammaln(cb + mb) - gammaln(cb))
    d = np.where(small, d, digamma(cb + mb) - digamma(cb))
    return l, d


def beta_terms(L, eta, phi):
    """(log p_i with every constant, d / d eta_i, d / d phi) of every observation of Beta likelihood L."""
    mu, mc, v = logit_parts(eta)
    a, b, w = phi * mu, phi * mc, phi * v
    y = np.asarray(L.y, dtype=np.float64)
    if L.dist == "beta_logit":
        ly, l1y = np.log(y), np.log1p(-y)
        ua, ub = ly - digamma(a), l1y - digamma(b)
        lp = gammaln(phi) - gammaln(a) - gammaln(b) + (a - 1.0) * ly + (b - 1.0) * l1y
        return lp, w * (ua - ub), digamma(phi) + mu * ua + mc * ub
    n = np.broadcast_to(np.asarray(L.trials, dtype=np.float64), y.shape)
    (la, da), (lb, db), (lf, df) = rising(a, y), rising(b, n - y), rising(phi, n)
    binomln = gammaln(n + 1.0) - gammaln(y + 1.0) - gammaln(n - y + 1.0)
    return binomln + la + lb - lf, w * (da - db), mu * da + mc * db - df


class BetaLogp:
    def __init__(self, ir: ModelIR, base=None):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()
        self.beta = [L for L in ir.likelihoods if L.dist in BETA_LIKS]
        self.base = (base or ir_numpy_mixture.make_logp)(
            dataclasses.replace(ir, likelihoods=[L for L in ir.likelihoods if L.dist not in BETA_LIKS]))

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def constrained(self, q):
        return ir_numpy_ordinal.OrdinalLogp.constrained(self, q)

    def eta(self, L, x):
        return ir_numpy_bounded.BoundedLogp.eta(self, L, x)

    def param(self, L, x):
        """(phi, its slot in x or None)."""
        if isinstance(L.phi, Ref):
            o = self.off[self.ir.var(L.phi.var).name]
            return x[o], o
        return float(L.phi), None

    def loglik(self, L, x):
        """log p(y_i | x) of every observation of likelihood L, with every constant."""
        return beta_terms(L, self.eta(L, x)[0], self.param(L, x)[0])[0]

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        lp, g = self.base(q)
        x, dxdq = self.constrained(q)
        gx = np.zeros(self.n)
        for L in self.beta:
            eta, parts = self.eta(L, x)
            phi, slot = self.param(L, x)
            lpi, r, ds = beta_terms(L, eta, phi)
            lp += float(np.sum(lpi))
            ir_numpy_zero_inflated.ZeroInflatedLogp._pull(self, gx, parts, r)
            if slot is not None:
                gx[slot] += np.sum(ds)
        return float(lp), np.asarray(g, dtype=np.float64) + gx * dxdq


def make_logp(ir: ModelIR, base=None):
    """ir_numpy_mixture.make_logp (or ``base``) for any model of the closed set, with Beta likelihoods."""
    if any(L.dist in BETA_LIKS for L in ir.likelihoods):
        return BetaLogp(ir, base)
    return (base or ir_numpy_mixture.make_logp)(ir)
