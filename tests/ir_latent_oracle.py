"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` that holds latent factors:
Normal / StudentT priors whose location is an ``ir.Linear`` predictor or whose scale is one constant per element
(``ir.is_latent``).

Everything else of the model is evaluated by oracle/ir_numpy_families.make_logp unchanged; this adds the latent priors on
top, restating the reference's densities at the lines oracle/ir_numpy.py cites (Normal continuous.py:526-527, StudentT
continuous.py:1936-1944).  The gradient goes to the prior's own variable, to a random scale, and through the location's
terms to every factor, pulled the way the likelihood branch of oracle/ir_numpy.py pulls it (``np.bincount`` for indexed
targets; ``X.T @ r`` for a design term).  Pinned by tests/test_ir_latent.py against a 40-digit mpmath reference and
central differences."""
from __future__ import annotations

import dataclasses

import numpy as np
from scipy.special import gammaln

from oracle import ir_numpy, ir_numpy_families
from pymc_b200.ir import LINEAR_PRIORS, Linear, ModelIR, Ref, Term, is_design, is_latent

HALF_LOG_2PI = ir_numpy.HALF_LOG_2PI


class LatentLogp:
    def __init__(self, m: ModelIR):
        m.validate()
        self.m, self.n, self.off = m, m.n, m.offsets()
        self.latent = [p for p in m.priors if is_latent(p)]
        self.base = ir_numpy_families.make_logp(dataclasses.replace(m, priors=[p for p in m.priors if not is_latent(p)]))

    def _sl(self, name):
        v = self.m.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def _location(self, p, N, x):
        """(mu[N], pull) with pull(r, gx) adding d/dx of sum_j r_j mu_j to gx."""
        a = p.params[LINEAR_PRIORS[p.dist][0]]
        terms = a.terms if isinstance(a, Linear) else [Term([(a.var, None)]) if isinstance(a, Ref) else Term([], coef=float(a))]
        mu, parts = np.zeros(N), []
        for t in terms:
            if is_design(t):  # X @ x
                X, s = np.asarray(t.coef, dtype=np.float64), self._sl(t.factors[0][0])
                mu += X @ x[s]
                parts.append(("design", X, s))
                continue
            coef = np.ones(N) if t.coef is None else np.broadcast_to(np.asarray(t.coef, dtype=np.float64), (N,))
            vals = []
            for vn, idx in t.factors:
                xv = x[self._sl(vn)]
                vals.append(np.broadcast_to(xv, (N,)) if (idx is None and xv.size == 1) else (xv if idx is None else xv[idx]))
            mu += coef * np.prod(vals, axis=0)
            parts.append(("term", coef, vals, t.factors))

        def pull(r, gx):
            for part in parts:
                if part[0] == "design":
                    _, X, s = part
                    gx[s] += X.T @ r
                    continue
                _, coef, vals, factors = part
                for k, (vn, idx) in enumerate(factors):
                    contrib = r * coef * np.prod([v for j, v in enumerate(vals) if j != k], axis=0)
                    s = self._sl(vn)
                    if idx is None and (s.stop - s.start) == 1:
                        gx[s] += contrib.sum()
                    elif idx is None:
                        gx[s] += contrib
                    else:
                        gx[s] += np.bincount(idx, weights=contrib, minlength=s.stop - s.start)
        return mu, pull

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        lp, g = self.base(q)
        x, dxdq = np.empty(self.n), np.ones(self.n)
        for v in self.m.vars:  # the constrained values, as ir_numpy computes them
            s = self._sl(v.name)
            if v.transform == "log":
                x[s] = np.exp(q[s])
                dxdq[s] = x[s]
            elif v.transform == "interval":
                lo, hi = v.bounds
                sg = ir_numpy._sigmoid(q[s])
                x[s] = lo + (hi - lo) * sg
                dxdq[s] = (hi - lo) * ir_numpy._dsigmoid(q[s])
            else:
                x[s] = q[s]
        gx = np.zeros(self.n)
        for p in self.latent:
            s = self._sl(p.var)
            xv, m = x[s], s.stop - s.start
            mu, pull = self._location(p, m, x)
            a = p.params[LINEAR_PRIORS[p.dist][1]]
            slot = self.off[self.m.var(a.var).name] if isinstance(a, Ref) else None
            sg = x[slot] if slot is not None else (np.asarray(a, dtype=np.float64) if np.ndim(a) else float(a))
            log_sg = np.broadcast_to(np.log(sg), (m,))
            z = (xv - mu) / sg
            if p.dist == "normal":  # continuous.py:526-527
                lp += float(np.sum(-0.5 * z * z - HALF_LOG_2PI - log_sg))
                r, rs = z / sg, (z * z - 1.0) / sg  # d/dmu, d/dsigma per element
            else:  # continuous.py:1936-1944
                nu = float(p.params[0])
                lp += float(np.sum(gammaln((nu + 1) / 2) - gammaln(nu / 2) - 0.5 * np.log(nu * np.pi) - log_sg
                                   - 0.5 * (nu + 1) * np.log1p(z * z / nu)))
                r = (nu + 1.0) * z / (sg * (nu + z * z))
                rs = -1.0 / sg + r * z
            gx[s] += -r
            pull(r, gx)
            if slot is not None:
                gx[slot] += np.sum(rs)
        return float(lp), g + gx * dxdq


def make_logp(m: ModelIR) -> LatentLogp:
    return LatentLogp(m)
