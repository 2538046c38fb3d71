"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` with ordered variables
(``Ordered`` transform, transforms.py:79-120) and ordinal likelihoods: ``ordered_logistic`` and ``ordered_probit``.

Layered like oracle/ir_numpy_bounded.py: the rest of the model is evaluated by the oracle it is given (by default
ir_numpy_bounded.make_logp; tests pass tests/ir_latent_oracle.make_logp for latent cutpoint priors) with each ordered
variable presented untransformed at its constrained value.  This module then adds the ordinal factors, the ordered
log-Jacobian and the chain rule through the cumulative sum.  The densities, as the Categorical they build
(Categorical.logp, discrete.py:1190-1206):

  ordered_logistic   OrderedLogistic.compute_p, discrete.py:1312-1326: p_y = sigmoid(c_y - eta) - sigmoid(c_{y-1} - eta)
  ordered_probit     OrderedProbit.compute_p, discrete.py:1416-1432: p_y = Phi((c_y - eta) / s) - Phi((c_{y-1} - eta) / s)

with c_{-1} = -inf and c_{K-1} = +inf, evaluated in log space: the logistic form as -softplus(-b) - softplus(a) +
log1mexp(a - b) with the gap from the cutpoints, the probit one by ir_numpy_bounded.log_mass.  Only real-line priors on an
ordered variable are evaluated (the base oracle sees it untransformed).

Pinned by tests/test_ir_ordinal.py against a 40-digit mpmath reference, scipy and central differences.  Only tests/ may
import it.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from oracle import ir_numpy, ir_numpy_bounded
from pymc_b200.ir import ORDERED_TRANSFORMS, ORDINAL_LIKS, ModelIR, Ref, ordered_backward

_softplus, _sigmoid = ir_numpy._softplus, ir_numpy._sigmoid


def ordinal_terms(dist, y, eta, s, c):
    """(log p_i, s d log p_i / d eta_i, w_i = d log p_i / d c_{y_i}, d log p_i / d s) of ordinal observations y (integers
    0..K-1) at linear predictor eta, scale s (1 for the logistic link) and cutpoints c (K - 1 of them)."""
    y = np.asarray(y).astype(np.int64)
    c = np.asarray(c, dtype=np.float64)
    K = len(c) + 1
    eta, s = np.broadcast_arrays(np.asarray(eta, dtype=np.float64), np.asarray(s, dtype=np.float64))
    lo_open, hi_open = y == 0, y == K - 1
    cl, ch = c[np.maximum(y - 1, 0)], c[np.minimum(y, K - 2)]
    a = np.where(lo_open, -np.inf, (cl - eta) / s)
    b = np.where(hi_open, np.inf, (ch - eta) / s)
    af, bf = np.where(lo_open, 0.0, a), np.where(hi_open, 0.0, b)  # an open side's finite stand-in (its terms are 0)
    if dist == "ordered_probit":
        lz, ra, rb = ir_numpy_bounded.log_mass(a, b)
        return lz, ra - rb, rb / s, (af * ra - bf * rb) / s
    mid = ~lo_open & ~hi_open
    gap = np.where(mid, (ch - cl) / s, 1.0)
    with np.errstate(divide="ignore"):
        lp = (np.where(lo_open, 0.0, -_softplus(af)) + np.where(hi_open, 0.0, -_softplus(-bf))
              + np.where(mid, np.log(-np.expm1(-gap)), 0.0))
    sa, sb = np.where(lo_open, 0.0, _sigmoid(af)), np.where(hi_open, 0.0, _sigmoid(-bf))
    w = sb + np.where(mid, 1.0 / np.expm1(gap), 0.0)
    return lp, sa - sb, w, np.zeros_like(lp)


class OrdinalLogp:
    def __init__(self, ir: ModelIR, base=None):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()
        self.ordinal = [L for L in ir.likelihoods if L.dist in ORDINAL_LIKS]
        self.ordered = [v for v in ir.vars if v.transform in ORDERED_TRANSFORMS]
        rest = dataclasses.replace(
            ir, vars=[dataclasses.replace(v, transform=None) if v.transform in ORDERED_TRANSFORMS else v for v in ir.vars],
            likelihoods=[L for L in ir.likelihoods if L.dist not in ORDINAL_LIKS])
        self.base = (base or ir_numpy_bounded.make_logp)(rest)

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def constrained(self, q):
        """(x, dx/dq) for the elementwise transforms; an ordered variable's x is its cumulative sum (dx/dq unused)."""
        x, dxdq = np.empty(self.n), np.ones(self.n)
        for v in self.ir.vars:
            s = self._sl(v.name)
            if v.transform == "log":
                x[s] = np.exp(q[s])
                dxdq[s] = x[s]
            elif v.transform == "interval":
                lo, hi = v.bounds
                x[s] = lo + (hi - lo) * _sigmoid(q[s])
                dxdq[s] = (hi - lo) * ir_numpy._dsigmoid(q[s])
            elif v.transform in ORDERED_TRANSFORMS:
                x[s] = ordered_backward(q[s].copy(), v.transform == "ordered_positive")
            else:
                x[s] = q[s]
        return x, dxdq

    def cutpoints(self, L, x):
        return x[self._sl(L.cutpoints.var)] if isinstance(L.cutpoints, Ref) else np.asarray(L.cutpoints, dtype=np.float64)

    def scale(self, L, x):
        """(s as a scalar or one per observation, its slot in x or None); 1 for the logistic link."""
        if L.dist == "ordered_logistic":
            return 1.0, None
        if isinstance(L.sigma, Ref):
            o = self.off[self.ir.var(L.sigma.var).name]
            return x[o], o
        return np.asarray(L.sigma, dtype=np.float64), None

    def eta(self, L, x):
        # the bounded oracle's predictor (every term kind, design terms included) over this model's layout
        return ir_numpy_bounded.BoundedLogp.eta(self, L, x)

    def loglik(self, L, x):
        """log p(y_i | x) of every observation of ordinal likelihood L (it has no constant)."""
        s, _ = self.scale(L, x)
        return ordinal_terms(L.dist, L.y, self.eta(L, x)[0], s, self.cutpoints(L, x))[0]

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        x, dxdq = self.constrained(q)
        qb = q.copy()
        for v in self.ordered:  # the base oracle sees the ordered variables untransformed, at their constrained values
            qb[self._sl(v.name)] = x[self._sl(v.name)]
        lp, g = self.base(qb)
        g = np.array(g, dtype=np.float64)
        gx = np.zeros(self.n)
        for L in self.ordinal:
            eta, parts = self.eta(L, x)
            s, slot = self.scale(L, x)
            lpi, rs, w, ds = ordinal_terms(L.dist, L.y, eta, s, self.cutpoints(L, x))
            lp += float(np.sum(lpi))
            r = rs / s
            if slot is not None:
                gx[slot] += np.sum(ds)
            if isinstance(L.cutpoints, Ref):  # d/dc_k: w over category k, -r - w over category k + 1
                y = np.asarray(L.y).astype(np.int64)
                K1 = self.ir.var(L.cutpoints.var).size
                up = y > 0
                gx[self._sl(L.cutpoints.var)] += (np.bincount(y, weights=w, minlength=K1 + 1)[:K1]
                                                  + np.bincount(y[up] - 1, weights=(-r - w)[up], minlength=K1)[:K1])
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
        out = g + gx * dxdq
        for v in self.ordered:  # log|J| and the chain rule through the cumulative sum (reverse cumsum, k descending)
            sl = self._sl(v.name)
            z = q[sl]
            pos = v.transform == "ordered_positive"
            lp += float(np.cumsum(z if pos else z[1:])[-1]) if (pos or v.size > 1) else 0.0
            S = np.cumsum((g[sl] + gx[sl])[::-1])[::-1]
            gq = np.exp(z) * S + 1.0
            if not pos:
                gq[0] = S[0]
            out[sl] = gq
        return float(lp), out


def make_logp(ir: ModelIR, base=None):
    """ir_numpy_bounded.make_logp (or ``base``) for any model of the closed set, with ordered variables and ordinal
    likelihoods."""
    if any(L.dist in ORDINAL_LIKS for L in ir.likelihoods) or any(v.transform in ORDERED_TRANSFORMS for v in ir.vars):
        return OrdinalLogp(ir, base)
    return (base or ir_numpy_bounded.make_logp)(ir)
