"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` whose likelihoods include the
count and positive families: ``binomial_logit``, ``negative_binomial_log`` and ``gamma_log``.

Everything else of the model (transforms and their Jacobians, priors, the other likelihoods, AR(1)) is evaluated by
oracle/ir_numpy.py unchanged; this module adds the three families on top, each restating the reference's density at the
line it cites, with the gradient with respect to eta (pulled through the linear predictor exactly as ir_numpy does) and,
for a random dispersion alpha, with respect to alpha through ``scipy.special.digamma``.

Pinned by tests/test_ir_families.py against ``scipy.stats`` (binom, nbinom, gamma), central differences and the
reference's own known answers.  Only tests/ and the golden generator may import this module.
"""
from __future__ import annotations

import dataclasses

import numpy as np
from scipy.special import digamma, gammaln

from oracle import ir_numpy
from pymc_b200.ir import NEGBIN_POISSON_ALPHA, ModelIR, Ref

FAMILIES = ("binomial_logit", "negative_binomial_log", "gamma_log")
_softplus, _sigmoid = ir_numpy._softplus, ir_numpy._sigmoid


def family_loglik(L, eta, a):
    """Per-observation log-likelihood of likelihood ``L`` at linear predictor ``eta`` and dispersion ``a`` (ignored by the
    binomial), with every constant included; what pm.compute_log_likelihood records."""
    y = np.asarray(L.y, dtype=np.float64)
    if L.dist == "binomial_logit":
        n = np.broadcast_to(np.asarray(L.trials, dtype=np.float64), y.shape)
        return gammaln(n + 1.0) - gammaln(y + 1.0) - gammaln(n - y + 1.0) + y * eta - n * _softplus(eta)
    if L.dist == "negative_binomial_log":
        if a > NEGBIN_POISSON_ALPHA:
            return y * eta - np.exp(eta) - gammaln(y + 1.0)
        d = eta - np.log(a)
        return gammaln(y + a) - gammaln(a) - gammaln(y + 1.0) - y * _softplus(-d) - a * _softplus(d)
    if L.dist == "gamma_log":
        return a * np.log(a) - a * eta - gammaln(a) + (a - 1.0) * np.log(y) - a * y * np.exp(-eta)
    raise NotImplementedError(L.dist)


class FamilyLogp:
    def __init__(self, ir: ModelIR):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()
        self.fam = [L for L in ir.likelihoods if L.dist in FAMILIES]
        self.base = ir_numpy.IrLogp(dataclasses.replace(ir, likelihoods=[L for L in ir.likelihoods if L.dist not in FAMILIES]))

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        lp, g = self.base(q)
        x, dxdq = np.empty(self.n), np.ones(self.n)
        for v in self.ir.vars:  # the constrained values, as ir_numpy computes them
            s = self._sl(v.name)
            if v.transform == "log":
                x[s] = np.exp(q[s])
                dxdq[s] = x[s]
            elif v.transform == "interval":
                lo, hi = v.bounds
                sg = _sigmoid(q[s])
                x[s] = lo + (hi - lo) * sg
                dxdq[s] = (hi - lo) * ir_numpy._dsigmoid(q[s])
            else:
                x[s] = q[s]
        gx = np.zeros(self.n)
        for L in self.fam:
            y = np.asarray(L.y, dtype=np.float64)
            N = len(y)
            eta = np.zeros(N)
            fvals = []
            for t in L.terms:
                coef = np.ones(N) if t.coef is None else np.broadcast_to(np.asarray(t.coef, dtype=np.float64), (N,))
                vals = []
                for vn, idx in t.factors:
                    xv = x[self._sl(vn)]
                    vals.append(np.broadcast_to(xv, (N,)) if (idx is None and xv.size == 1) else (xv if idx is None else xv[idx]))
                fvals.append((coef, vals))
                eta += coef * np.prod(vals, axis=0)
            a, slot = None, None
            if L.dist != "binomial_logit":
                if isinstance(L.alpha, Ref):
                    slot = self.off[self.ir.var(L.alpha.var).name]
                    a = x[slot]
                else:
                    a = float(L.alpha)
            lp += float(np.sum(family_loglik(L, eta, a)))
            if L.dist == "binomial_logit":
                # discrete.py:141-152: binomln(n, y) + y log p + (n - y) log(1 - p), p = sigmoid(eta); in PyTensor's
                # stabilised log-sigmoid forms binomln(n, y) + y eta - n softplus(eta)
                n = np.broadcast_to(np.asarray(L.trials, dtype=np.float64), (N,))
                r = y - n * _sigmoid(eta)
            elif L.dist == "negative_binomial_log":
                # discrete.py:700-745, n = a, p = a / (mu + a), mu = exp(eta):
                #   lgamma(y + a) - lgamma(a) - lgamma(y + 1) + y (eta - lse) + a (log a - lse),  lse = logaddexp(eta, log a)
                # and the Poisson(mu) limit above a = 1e10 (discrete.py:727-735), whose alpha gradient is 0
                if a > NEGBIN_POISSON_ALPHA:
                    r = y - np.exp(eta)
                else:
                    d = eta - np.log(a)
                    s, sc = _sigmoid(d), _sigmoid(-d)  # mu / (mu + a), a / (mu + a)
                    r = y * sc - a * s  # a (y - mu) / (mu + a)
                    if slot is not None:  # psi(y + a) - psi(a) + log a + 1 - lse - (y + a) / (mu + a)
                        gx[slot] += np.sum(digamma(y + a) - digamma(a) + 1.0 - _softplus(d) - sc * (1.0 + y / a))
            else:
                # continuous.py:2512-2521 with beta = a exp(-eta): a log a - a eta - lgamma(a) + (a - 1) log y - a y exp(-eta)
                w = y * np.exp(-eta)
                r = a * (w - 1.0)
                if slot is not None:  # log a + 1 - eta - psi(a) + log y - y exp(-eta)
                    gx[slot] += np.sum(np.log(a) + 1.0 - eta - digamma(a) + np.log(y) - w)
            for t, (coef, vals) in zip(L.terms, fvals):
                for k, (vn, idx) in enumerate(t.factors):
                    others = coef * np.prod([v for j, v in enumerate(vals) if j != k], axis=0) if len(vals) > 1 else coef
                    s = self._sl(vn)
                    contrib = r * others
                    if idx is None and (s.stop - s.start) == 1:
                        gx[s] += contrib.sum()
                    elif idx is None:
                        gx[s] += contrib
                    else:
                        gx[s] += np.bincount(idx, weights=contrib, minlength=s.stop - s.start)
        return float(lp), g + gx * dxdq


def make_logp(ir: ModelIR):
    """ir_numpy.make_logp for any model of the closed set, including the three families above."""
    return FamilyLogp(ir) if any(L.dist in FAMILIES for L in ir.likelihoods) else ir_numpy.make_logp(ir)
