"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` whose likelihoods include
Normal observations measured with bounds: ``censored_normal`` and ``truncated_normal``.

Everything else of the model (transforms and their Jacobians, priors, the other likelihoods) is evaluated by
oracle/ir_numpy_families.py unchanged; this module adds the two factors on top, with the gradient with respect to eta
(pulled through every term kind, design terms included) and with respect to a random sigma.  The densities:

  censored_normal    logprob/censoring.py:213-248 over Normal (continuous.py:526-546): log Phi(z) where y_i == lower_i
                     (normal_lcdf, dist_math.py:126-133), log(1 - Phi(z)) where y_i == upper_i (normal_lccdf, :136-142),
                     the Normal log-density elsewhere; z = (y_i - eta_i) / sigma
  truncated_normal   TruncatedNormal.logp, continuous.py:720-747: the Normal log-density minus log Z,
                     Z = Phi(beta) - Phi(alpha) of the standardised bounds (log_diff_normal_cdf, dist_math.py:145-182),
                     1 - Phi(alpha) with only a lower bound, Phi(beta) with only an upper one

The log-CDFs are scipy.special.log_ndtr.  The gradients need phi / Phi and phi / Z: these ratios are formed from erfcx()
with the common Gaussian factor cancelled, so a window far in a tail keeps its accuracy.

Pinned by tests/test_ir_bounded.py against a 40-digit mpmath reference and scipy.stats.  Only tests/ may import it.
"""
from __future__ import annotations

import dataclasses

import numpy as np
from scipy.special import erf, erfcx, log_ndtr

from oracle import ir_numpy_families
from pymc_b200.ir import BOUNDED_LIKS, ModelIR, Ref, is_design

HALF_LOG_2PI = 0.5 * np.log(2.0 * np.pi)
SQRT_2_PI = np.sqrt(2.0 / np.pi)
SQRT_HALF = np.sqrt(0.5)


def mills(z):
    """phi(z) / Phi(z), elementwise."""
    z = np.asarray(z, dtype=np.float64)
    with np.errstate(over="ignore", under="ignore"):
        return np.where(z < -1.0, SQRT_2_PI / erfcx(-z * SQRT_HALF),
                        np.exp(-0.5 * z * z - HALF_LOG_2PI - log_ndtr(np.maximum(z, -1.0))))


def log_mass(a, b):
    """(log Z, phi(a) / Z, phi(b) / Z) with Z = Phi(b) - Phi(a), elementwise, a < b; a = -inf / b = +inf for an open side."""
    a, b = np.broadcast_arrays(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64))
    lz, ra, rb = np.zeros(a.shape), np.zeros(a.shape), np.zeros(a.shape)
    lo_open, hi_open = np.isneginf(a), np.isposinf(b)
    k = lo_open & ~hi_open  # upper bound only: Phi(b)
    lz[k], rb[k] = log_ndtr(b[k]), mills(b[k])
    k = hi_open & ~lo_open  # lower bound only: 1 - Phi(a)
    lz[k], ra[k] = log_ndtr(-a[k]), mills(-a[k])
    two = ~lo_open & ~hi_open
    for k, flip in ((two & (a > 0), True), (two & (b < 0), False)):
        # one tail: with t = the bound nearer the mode and f the farther one (mirrored into the lower tail),
        # Z = Phi(t) (1 - Phi(f) / Phi(t)), Phi(f) / Phi(t) = exp((t - f)(t + f) / 2) erfcx(-f / sqrt 2) / erfcx(-t / sqrt 2)
        t, f = (-a[k], -b[k]) if flip else (b[k], a[k])
        rho = np.exp(0.5 * (t - f) * (t + f)) * erfcx(-f * SQRT_HALF) / erfcx(-t * SQRT_HALF)
        lz[k] = log_ndtr(t) + np.log1p(-rho)
        r_near = mills(t) / (1.0 - rho)      # phi(t) / Z
        r_far = r_near * rho * mills(f) / mills(t)  # phi(f) / Z = (phi(f) / Phi(f)) (Phi(f) / Phi(t)) Phi(t) / Z
        if flip:
            ra[k], rb[k] = r_near, r_far
        else:
            rb[k], ra[k] = r_near, r_far
    k = two & (a <= 0) & (b >= 0)  # the window holds the mode: no cancellation
    w = 0.5 * (erf(b[k] * SQRT_HALF) - erf(a[k] * SQRT_HALF))
    lz[k] = np.log(w)
    ra[k] = np.exp(-0.5 * a[k] ** 2 - HALF_LOG_2PI) / w
    rb[k] = np.exp(-0.5 * b[k] ** 2 - HALF_LOG_2PI) / w
    return lz, ra, rb


def censor_codes(L):
    """0: observed; 1: at its lower bound; 2: at its upper bound."""
    y = np.asarray(L.y, dtype=np.float64)
    lo, hi = L.bounds()
    return np.where(y == lo, 1, np.where(y == hi, 2, 0))


def bounded_loglik(L, eta, sg):
    """Per-observation log-likelihood with every constant; what pm.compute_log_likelihood records."""
    y = np.asarray(L.y, dtype=np.float64)
    z = (y - eta) / sg
    normal = -0.5 * z * z - HALF_LOG_2PI - np.log(sg) * np.ones_like(z)
    if L.dist == "censored_normal":
        c = censor_codes(L)
        return np.where(c == 1, log_ndtr(z), np.where(c == 2, log_ndtr(-z), normal))
    lo, hi = L.bounds()
    return normal - log_mass((lo - eta) / sg, (hi - eta) / sg)[0]


def _bounded_grad(L, eta, sg):
    """(d loglik_i / d eta_i, d loglik_i / d sigma)."""
    y = np.asarray(L.y, dtype=np.float64)
    z = (y - eta) / sg
    if L.dist == "censored_normal":
        c = censor_codes(L)
        zc = np.where(c == 2, -z, z)  # log(1 - Phi(z)) = log Phi(-z)
        lam = mills(zc)
        r = np.where(c == 0, z / sg, np.where(c == 1, -lam, lam) / sg)
        ds = np.where(c == 0, (z * z - 1.0) / sg, -lam * zc / sg)
        return r, ds
    lo, hi = L.bounds()
    a, b = (lo - eta) / sg, (hi - eta) / sg
    _, ra, rb = log_mass(a, b)
    ta = np.where(np.isinf(a), 0.0, a) * ra  # an open side: phi(-inf) = 0, -inf * 0 = 0
    tb = np.where(np.isinf(b), 0.0, b) * rb
    return (z + rb - ra) / sg, (z * z - 1.0 + tb - ta) / sg


class BoundedLogp:
    def __init__(self, ir: ModelIR):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()
        self.bounded = [L for L in ir.likelihoods if L.dist in BOUNDED_LIKS]
        self.base = ir_numpy_families.make_logp(
            dataclasses.replace(ir, likelihoods=[L for L in ir.likelihoods if L.dist not in BOUNDED_LIKS]))

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def constrained(self, q):
        """(x, dx/dq) as ir_numpy computes them."""
        x, dxdq = np.empty(self.n), np.ones(self.n)
        for v in self.ir.vars:
            s = self._sl(v.name)
            if v.transform == "log":
                x[s] = np.exp(q[s])
                dxdq[s] = x[s]
            elif v.transform == "interval":
                lo, hi = v.bounds
                x[s] = lo + (hi - lo) * ir_numpy_families._sigmoid(q[s])
                dxdq[s] = (hi - lo) * ir_numpy_families.ir_numpy._dsigmoid(q[s])
            else:
                x[s] = q[s]
        return x, dxdq

    def eta(self, L, x):
        """The linear predictor and, per term, what its gradient needs."""
        N = len(L.y)
        eta, parts = np.zeros(N), []
        for t in L.terms:
            if is_design(t):
                X = np.asarray(t.coef, dtype=np.float64)
                s = self._sl(t.factors[0][0])
                eta += X @ x[s]
                parts.append(("design", X, s))
                continue
            coef = np.ones(N) if t.coef is None else np.broadcast_to(np.asarray(t.coef, dtype=np.float64), (N,))
            vals = []
            for vn, idx in t.factors:
                xv = x[self._sl(vn)]
                vals.append(np.broadcast_to(xv, (N,)) if (idx is None and xv.size == 1) else (xv if idx is None else xv[idx]))
            eta += coef * np.prod(vals, axis=0)
            parts.append(("terms", coef, vals, t))
        return eta, parts

    def sigma(self, L, x):
        """(sigma as a scalar or one per observation, its slot in x or None)."""
        if isinstance(L.sigma, Ref):
            o = self.off[self.ir.var(L.sigma.var).name]
            return x[o], o
        return np.asarray(L.sigma, dtype=np.float64), None

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        lp, g = self.base(q)
        x, dxdq = self.constrained(q)
        gx = np.zeros(self.n)
        for L in self.bounded:
            eta, parts = self.eta(L, x)
            sg, slot = self.sigma(L, x)
            lp += float(np.sum(bounded_loglik(L, eta, sg)))
            r, ds = _bounded_grad(L, eta, sg)
            if slot is not None:
                gx[slot] += np.sum(ds)
            for p in parts:
                if p[0] == "design":
                    _, X, s = p
                    gx[s] += X.T @ r
                    continue
                _, coef, vals, t = p
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
    """ir_numpy_families.make_logp for any model of the closed set, including the two bounded Normal likelihoods."""
    return BoundedLogp(ir) if any(L.dist in BOUNDED_LIKS for L in ir.likelihoods) else ir_numpy_families.make_logp(ir)
