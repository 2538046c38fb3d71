"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` with survival likelihoods
(``SURVIVAL_LIKS``): ``weibull_log`` and ``lognormal``, plain, censored or truncated.

Layered like oracle/ir_numpy_zero_inflated.py: the rest of the model (every other factor, the priors of alpha / sigma and
every transform) is evaluated by the oracle it is given (by default ir_numpy_zero_inflated.make_logp, which covers every
other factor of the closed set).  This module adds the survival factors with every constant:

  weibull_log    Weibull(alpha, beta = e^eta), continuous.py:2740-2831, with u = log y - eta and t = e^{alpha u}:
                 log f = log alpha - eta + (alpha - 1) u - t;  log S = -t;  log F = log(1 - e^-t)
                 (log t - t / 2 below t = 2e-9, where 1 - e^-t has lost its digits or underflowed)
  lognormal      LogNormal(eta, sigma), continuous.py:1723-1846: the Normal of log y, minus log y where there is a density;
                 its censored / truncated forms are ir_numpy_bounded's Normal ones on log y and log bounds
  censored       logprob/censoring.py:213-248: log F(y) where y_i == lower_i, log S(y) where y_i == upper_i
  truncated      the density minus log(S(lower) - S(upper)); for the Weibull e^{-tA} (1 - e^{-D}), D = tB - tA formed as
                 log D = alpha uB + log(1 - e^{-alpha log(B / A)}), log(B / A) = log1p((B - A) / A)

A lower bound of 0 or -inf is an open side.  Pinned by tests/test_ir_survival.py against a 40-digit mpmath reference
(itself checked against scipy.stats) and central differences.  Only tests/ may import it.
"""
from __future__ import annotations

import dataclasses
import types

import numpy as np

from oracle import ir_numpy_bounded, ir_numpy_ordinal, ir_numpy_zero_inflated
from pymc_b200.ir import LOGNORMAL_LIKS, SURVIVAL_LIKS, WEIBULL_LIKS, ModelIR, Ref


def _log1mexp_neg(v, t):
    """log(1 - e^-t) given v = log t."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return np.where(v < -20.0, v - 0.5 * t, np.where(t < np.log(2.0), np.log(-np.expm1(-t)), np.log1p(-np.exp(-t))))


def _t_over_expm1(v, t):
    """t / (e^t - 1) given v = log t."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return np.where(v < -20.0, 1.0 - 0.5 * t, np.where(v > 700.0, 0.0, t / np.expm1(t)))


def censor_codes(L):
    """0: observed (or not a censored likelihood); 1: at its lower bound; 2: at its upper bound."""
    y = np.asarray(L.y, dtype=np.float64)
    if not L.dist.startswith("censored"):
        return np.zeros(len(y), dtype=int)
    lo, hi = L.bounds()
    return np.where(y == lo, 1, np.where(y == hi, 2, 0))


def weibull_terms(L, eta, a):
    """(log p_i, d / d eta_i, d / d alpha) of every Weibull observation."""
    y = np.asarray(L.y, dtype=np.float64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        u = np.log(y) - eta
        v = a * u
        t = np.exp(v)
        c = censor_codes(L)
        q = _t_over_expm1(v, t)
        lp = np.where(c == 2, -t, np.where(c == 1, _log1mexp_neg(v, t), np.log(a) - eta + (a - 1.0) * u - t))
        r = np.where(c == 2, a * t, np.where(c == 1, -a * q, a * (t - 1.0)))
        s = np.where(c == 2, -u * t, np.where(c == 1, u * q, 1.0 / a + u - u * t))
        if L.dist == "truncated_weibull_log":
            lo, hi = L.bounds()
            A = np.where(lo > 0, lo, 0.0)
            has_a, has_b = A > 0, np.isfinite(hi)
            ua = np.where(has_a, np.log(np.where(has_a, A, 1.0)) - eta, 0.0)
            ta = np.where(has_a, np.exp(a * ua), 0.0)
            lp, r, s = lp + ta, r - a * ta, s + ua * ta
            ub = np.log(np.where(has_b, hi, 1.0)) - eta
            lr = np.where(has_a & has_b, np.log1p((np.where(has_b, hi, 1.0) - A) / np.where(has_a, A, 1.0)), 0.0)
            ld = np.where(has_a, a * ub + np.log(-np.expm1(-a * np.where(has_a, lr, 1.0))), a * ub)
            d = np.exp(ld)
            qd = _t_over_expm1(ld, d)
            tail = np.where(has_a, lr / np.expm1(a * np.where(has_a, lr, 1.0)), 0.0)
            lp = np.where(has_b, lp - _log1mexp_neg(ld, d), lp)
            r = np.where(has_b, r + a * qd, r)
            s = np.where(has_b, s - qd * (ub + tail), s)
    return lp, r, s


def _as_normal(L):
    """The censored / truncated Normal on log y and log bounds that a LogNormal likelihood is, as ir_numpy_bounded reads it
    (a plain one: censored with open sides).  The censoring codes are those of y itself."""
    y = np.asarray(L.y, dtype=np.float64)
    lo, hi = L.bounds()
    c = censor_codes(L)
    with np.errstate(divide="ignore"):
        llo = np.where(c == 1, np.log(y), np.where(lo > 0, np.log(np.where(lo > 0, lo, 1.0)), -np.inf))
        lhi = np.where(c == 2, np.log(y), np.log(hi))
    dist = "truncated_normal" if L.dist == "truncated_lognormal" else "censored_normal"
    return types.SimpleNamespace(dist=dist, y=np.log(y), bounds=lambda: (llo, lhi))


def lognormal_terms(L, eta, sg):
    """(log p_i, d / d eta_i, d / d sigma) of every LogNormal observation."""
    N = _as_normal(L)
    lp = ir_numpy_bounded.bounded_loglik(N, eta, sg) - np.where(censor_codes(L) == 0, N.y, 0.0)
    r, ds = ir_numpy_bounded._bounded_grad(N, eta, sg)
    return lp, r, ds


def survival_terms(L, eta, par):
    """(log p_i with every constant, d / d eta_i, d / d alpha or sigma) of every observation."""
    return weibull_terms(L, eta, par) if L.dist in WEIBULL_LIKS else lognormal_terms(L, eta, par)


class SurvivalLogp:
    def __init__(self, ir: ModelIR, base=None):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()
        self.surv = [L for L in ir.likelihoods if L.dist in SURVIVAL_LIKS]
        self.base = (base or ir_numpy_zero_inflated.make_logp)(
            dataclasses.replace(ir, likelihoods=[L for L in ir.likelihoods if L.dist not in SURVIVAL_LIKS]))

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def constrained(self, q):
        return ir_numpy_ordinal.OrdinalLogp.constrained(self, q)

    def eta(self, L, x):
        return ir_numpy_bounded.BoundedLogp.eta(self, L, x)

    def param(self, L, x):
        """(alpha of a Weibull or sigma of a LogNormal, a scalar or one per observation; its slot in x or None)."""
        p = L.sigma if L.dist in LOGNORMAL_LIKS else L.alpha
        if isinstance(p, Ref):
            o = self.off[self.ir.var(p.var).name]
            return x[o], o
        return np.asarray(p, dtype=np.float64), None

    def loglik(self, L, x):
        """log p(y_i | x) of every observation of likelihood L, with every constant."""
        return survival_terms(L, self.eta(L, x)[0], self.param(L, x)[0])[0]

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        lp, g = self.base(q)
        x, dxdq = self.constrained(q)
        gx = np.zeros(self.n)
        for L in self.surv:
            eta, parts = self.eta(L, x)
            par, slot = self.param(L, x)
            lpi, r, ds = survival_terms(L, eta, par)
            lp += float(np.sum(lpi))
            ir_numpy_zero_inflated.ZeroInflatedLogp._pull(self, gx, parts, r)
            if slot is not None:
                gx[slot] += np.sum(ds)
        return float(lp), np.asarray(g, dtype=np.float64) + gx * dxdq


def make_logp(ir: ModelIR, base=None):
    """ir_numpy_zero_inflated.make_logp (or ``base``) for any model of the closed set, with survival likelihoods."""
    if any(L.dist in SURVIVAL_LIKS for L in ir.likelihoods):
        return SurvivalLogp(ir, base)
    return (base or ir_numpy_zero_inflated.make_logp)(ir)
