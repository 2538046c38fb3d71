"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` with zero-inflated and
hurdle likelihoods (``ZI_LIKS``): ``zero_inflated_poisson`` / ``_binomial`` / ``_negative_binomial``, ``hurdle_poisson`` /
``_negative_binomial`` / ``_gamma``.

Layered like oracle/ir_numpy_ordinal.py: the rest of the model (every other factor, the psi variable's prior and every
transform) is evaluated by the oracle it is given (by default ir_numpy_ordinal.make_logp).  This module adds the
zero-inflated and hurdle factors with every constant, as the reference writes them (pymc/distributions/mixture.py):

  zero-inflated  mixture_logprob, :470-494, a logsumexp over [DiracDelta(0), f] with weights [1 - psi, psi]:
                 y = 0: logaddexp(log(1 - psi), log psi + log P0);  y > 0: log psi + log f(y)
  hurdle         marginal_hurdle_logprob, :847-870, with f = Truncated(f, lower=1) for the counts (:826-829):
                 y = 0: log(1 - psi);  y > 0: log psi + log f(y) - log(1 - P0)  (hurdle_gamma: log psi + log f(y))

f is the family of ``ZI_FAMILY`` at eta (ir_numpy_families' forms), P0 = f(0).  psi is a constant, a scalar variable or
sigmoid(zeta) of a Linear zeta, with log psi = -softplus(-zeta) and log(1 - psi) = -softplus(zeta).

Pinned by tests/test_ir_zero_inflated.py against a 40-digit mpmath reference (itself checked against scipy.stats
compositions) and central differences.  Only tests/ may import it.
"""
from __future__ import annotations

import dataclasses
import types

import numpy as np
from scipy.special import digamma, gammaln

from oracle import ir_numpy, ir_numpy_bounded, ir_numpy_ordinal
from pymc_b200.ir import NEGBIN_POISSON_ALPHA, ZI_FAMILY, ZI_LIKS, Linear, ModelIR, Ref

_softplus, _sigmoid = ir_numpy._softplus, ir_numpy._sigmoid


def _log1mexp(t):
    """log(1 - e^t) for t < 0."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(t > -np.log(2.0), np.log(-np.expm1(t)), np.log1p(-np.exp(t)))


def family_parts(dist, y, eta, nt, a):
    """(lf, rf, af, lP0, r0, a0, lm): log f(y) with every constant and its eta / alpha derivatives, log P0 = log f(0) with
    its derivatives, and lm = log(-log P0), of the family of ``dist``."""
    fam = ZI_FAMILY[dist]
    y, eta = np.asarray(y, dtype=np.float64), np.asarray(eta, dtype=np.float64)
    z = np.zeros_like(eta)
    if fam == "gamma_log":  # continuous.py:2512-2521, beta = a exp(-eta); at y = 0 a stand-in y (unused)
        ys = np.where(y > 0, y, 1.0)
        w = ys * np.exp(-eta)
        lf = a * np.log(a) - a * eta - gammaln(a) + (a - 1.0) * np.log(ys) - a * w
        af = np.log(a) + 1.0 - eta - digamma(a) + np.log(ys) - w
        return lf, a * (w - 1.0), af, z - np.inf, z, z, z + np.inf
    if fam == "binomial_logit":  # discrete.py:141-152
        n = np.broadcast_to(np.asarray(nt, dtype=np.float64), y.shape)
        lP0 = -n * _softplus(eta)
        lf = gammaln(n + 1.0) - gammaln(y + 1.0) - gammaln(n - y + 1.0) + y * eta + lP0
        r0 = -n * _sigmoid(eta)
        return lf, y + r0, z, lP0, r0, z, z + np.inf
    if fam == "negative_binomial_log" and a <= NEGBIN_POISSON_ALPHA:  # discrete.py:700-745
        d = eta - np.log(a)
        s, sc, sp = _sigmoid(d), _sigmoid(-d), _softplus(d)
        lP0 = -a * sp
        lf = gammaln(y + a) - gammaln(a) - gammaln(y + 1.0) - y * _softplus(-d) + lP0
        af = digamma(y + a) - digamma(a) + 1.0 - sp - sc * (1.0 + y / a)
        with np.errstate(divide="ignore"):
            lm = np.log(a) + np.where(d < -30.0, d - 0.5 * np.exp(np.minimum(d, 0.0)), np.log(sp))
        return lf, y * sc - a * s, af, lP0, -a * s, s - sp, lm
    mu = np.exp(eta)  # discrete.py:581-586, and the NegativeBinomial's Poisson limit (:727-735)
    return y * eta - mu - gammaln(y + 1.0), y - mu, z, -mu, -mu, z, eta


def zi_terms(dist, y, eta, nt, a, lpsi, l1psi, psi):
    """(log p_i, d/d eta_i, d/d zeta_i, d/d psi, d/d alpha) of every observation, psi being sigmoid(zeta) for the zeta
    derivative and the value itself for the psi derivative."""
    y = np.asarray(y, dtype=np.float64)
    lf, rf, af, lP0, r0, a0, lm = family_parts(dist, y, eta, nt, a)
    lpsi, l1psi, psi = (np.broadcast_to(np.asarray(v, dtype=np.float64), y.shape) for v in (lpsi, l1psi, psi))
    zero = y == 0
    if dist.startswith("hurdle"):
        lp0, r_0, dz0, dpsi0, da0 = l1psi, 0.0 * y, -psi, -np.exp(-l1psi), 0.0 * y
        lp1, r1, da1 = lpsi + lf, rf, af
        if dist != "hurdle_gamma":  # - log(1 - P0); log m where m = -log P0 < 1e-304
            tiny = lm < -700.0
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                q = np.where(tiny, 0.0, 1.0 / np.expm1(-lP0))
                lp1 = lp1 - np.where(tiny, lm, _log1mexp(lP0))
            r1 = np.where(tiny, r1 - 1.0, r1 + r0 * q)
            da1 = np.where(tiny, da1, da1 + a0 * q)
    else:
        t = lpsi + lP0
        u = t - l1psi
        lp0 = np.logaddexp(l1psi, t)
        w = _sigmoid(u)
        r_0, dz0, dpsi0, da0 = w * r0, w - psi, np.expm1(lP0) * np.exp(-lp0), w * a0
        lp1, r1, da1 = lpsi + lf, rf, af
    return (np.where(zero, lp0, lp1), np.where(zero, r_0, r1), np.where(zero, dz0, 1.0 - psi),
            np.where(zero, dpsi0, np.exp(-lpsi)), np.where(zero, da0, da1))


class ZeroInflatedLogp:
    def __init__(self, ir: ModelIR, base=None):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()
        self.zi = [L for L in ir.likelihoods if L.dist in ZI_LIKS]
        self.base = (base or ir_numpy_ordinal.make_logp)(
            dataclasses.replace(ir, likelihoods=[L for L in ir.likelihoods if L.dist not in ZI_LIKS]))

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def constrained(self, q):
        return ir_numpy_ordinal.OrdinalLogp.constrained(self, q)

    def eta(self, L, x):
        return ir_numpy_bounded.BoundedLogp.eta(self, L, x)

    def psi(self, L, x):
        """(log psi, log(1 - psi), psi, zeta parts or None, psi slot or None)."""
        if isinstance(L.psi, Linear):
            zeta, parts = self.eta(types.SimpleNamespace(y=L.y, terms=L.psi.terms), x)
            return -_softplus(-zeta), -_softplus(zeta), _sigmoid(zeta), parts, None
        if isinstance(L.psi, Ref):
            o = self.off[self.ir.var(L.psi.var).name]
            p, slot = x[o], o
        else:
            p, slot = float(L.psi), None
        return np.log(p), np.log1p(-p), p, None, slot

    def family_params(self, L, x):
        """(trials, alpha, alpha slot or None)."""
        fam = ZI_FAMILY[L.dist]
        if fam == "binomial_logit":
            return np.asarray(L.trials, dtype=np.float64), None, None
        if fam == "poisson_log":
            return None, None, None
        if isinstance(L.alpha, Ref):
            o = self.off[self.ir.var(L.alpha.var).name]
            return None, x[o], o
        return None, float(L.alpha), None

    def terms(self, L, x):
        nt, a, _ = self.family_params(L, x)
        lpsi, l1psi, p, _, _ = self.psi(L, x)
        return zi_terms(L.dist, L.y, self.eta(L, x)[0], nt, a, lpsi, l1psi, p)

    def loglik(self, L, x):
        """log p(y_i | x) of every observation of likelihood L, with every constant."""
        return self.terms(L, x)[0]

    def _pull(self, gx, parts, r):
        for p in parts:
            if p[0] == "design":
                _, X, sl = p
                gx[sl] += X.T @ r
                continue
            _, coef, vals, t = p
            for k, (vn, idx) in enumerate(t.factors):
                others = coef * np.prod([v for j, v in enumerate(vals) if j != k], axis=0) if len(vals) > 1 else coef
                sl = self._sl(vn)
                contrib = r * others
                if idx is None and (sl.stop - sl.start) == 1:
                    gx[sl] += contrib.sum()
                elif idx is None:
                    gx[sl] += contrib
                else:
                    gx[sl] += np.bincount(idx, weights=contrib, minlength=sl.stop - sl.start)

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        lp, g = self.base(q)
        x, dxdq = self.constrained(q)
        gx = np.zeros(self.n)
        for L in self.zi:
            eta, parts = self.eta(L, x)
            nt, a, aslot = self.family_params(L, x)
            lpsi, l1psi, p, zparts, pslot = self.psi(L, x)
            lpi, r, dz, dpsi, da = zi_terms(L.dist, L.y, eta, nt, a, lpsi, l1psi, p)
            lp += float(np.sum(lpi))
            self._pull(gx, parts, r)
            if zparts is not None:
                self._pull(gx, zparts, dz)
            if pslot is not None:
                gx[pslot] += np.sum(dpsi)
            if aslot is not None:
                gx[aslot] += np.sum(da)
        return float(lp), np.asarray(g, dtype=np.float64) + gx * dxdq


def make_logp(ir: ModelIR, base=None):
    """ir_numpy_ordinal.make_logp (or ``base``) for any model of the closed set, with zero-inflated and hurdle
    likelihoods."""
    if any(L.dist in ZI_LIKS for L in ir.likelihoods):
        return ZeroInflatedLogp(ir, base)
    return (base or ir_numpy_ordinal.make_logp)(ir)
