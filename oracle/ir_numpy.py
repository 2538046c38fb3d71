"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation of a ``pymc_b200.ir.ModelIR``: q -> (logp, dlogp).

The generic counterpart of oracle/logp_numpy.py: the same published density formulas (each citing the reference line it
follows), composed the way the reference composes a model's joint log-density:

  * every value variable is mapped to its constrained value and contributes the log-Jacobian of its transform
    (LogTransform pymc/logprob/transforms.py:880-891; IntervalTransform :1026-1073);
  * factors are summed with no reweighting (pymc/model/core.py:688-690);
  * the gradient is the chain rule through the transforms (what ``pytensor.grad`` of that graph produces,
    pymc/model/core.py:239-248).

Pinned by tests/test_ir.py: the IR forms of Eight Schools, Radon and stochastic volatility equal the hand-derived
restatements of oracle/logp_numpy.py (themselves pinned against scipy.stats and finite differences) to rounding, and
every density in the closed set is checked against ``scipy.stats`` and central differences.

Only tests/, bench.py's cpu_baseline leg and __graft_entry__.smoke() may import this module.
"""
from __future__ import annotations

import numpy as np
from scipy.special import gammaln

from pymc_b200.ir import ModelIR, Ref

HALF_LOG_2PI = 0.5 * np.log(2.0 * np.pi)


def _softplus(x):
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def _sigmoid(x):
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, 1.0 / (1.0 + e), e / (1.0 + e))


def _dsigmoid(x):
    """sigmoid(x) (1 - sigmoid(x)) as e / (1 + e)^2, e = exp(-|x|): no cancellation in 1 - sigmoid(x) at large |x|."""
    e = np.exp(-np.abs(x))
    return e / ((1.0 + e) * (1.0 + e))


class IrLogp:
    def __init__(self, ir: ModelIR):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def _par(self, a, x):
        """(value, slot or None): a constant, or the constrained value of a scalar variable."""
        if isinstance(a, Ref):
            o = self.off[self.ir.var(a.var).name]
            return x[o], o
        return float(a), None

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        ir, off = self.ir, self.off
        x = np.empty(self.n)
        dxdq = np.ones(self.n)
        djdq = np.zeros(self.n)
        lp = 0.0
        for v in ir.vars:
            s = slice(off[v.name], off[v.name] + v.size)
            if v.transform == "log":  # transforms.py:880-891: x = exp(z), log|J| = z
                x[s] = np.exp(q[s])
                dxdq[s] = x[s]
                djdq[s] = 1.0
                lp += q[s].sum()
            elif v.transform == "interval":  # transforms.py:1026-1073: x = lo + (hi-lo) sigmoid(z)
                lo, hi = v.bounds
                sg = _sigmoid(q[s])
                x[s] = lo + (hi - lo) * sg
                dxdq[s] = (hi - lo) * _dsigmoid(q[s])
                djdq[s] = 1.0 - 2.0 * sg
                lp += np.sum(np.log(hi - lo) - _softplus(-q[s]) - _softplus(q[s]))
            else:
                x[s] = q[s]
        gx = np.zeros(self.n)

        def add(slot, val):
            if slot is not None:
                gx[slot] += val

        # ---- priors ------------------------------------------------------------------------------------------------
        for p in ir.priors:
            s = self._sl(p.var)
            xv = x[s]
            m = xv.size
            d = p.dist
            if d == "flat":
                continue
            if d == "normal":  # continuous.py:526-527
                mu, smu = self._par(p.params[0], x)
                sg, ssg = self._par(p.params[1], x)
                z = (xv - mu) / sg
                lp += np.sum(-0.5 * z * z) - m * (HALF_LOG_2PI + np.log(sg))
                gx[s] += -z / sg
                add(smu, np.sum(z) / sg)
                add(ssg, np.sum(z * z - 1.0) / sg)
            elif d == "halfnormal":  # continuous.py:909-911
                sg, ssg = self._par(p.params[0], x)
                z = xv / sg
                lp += np.sum(-0.5 * z * z) + m * (0.5 * np.log(2.0 / np.pi) - np.log(sg))
                gx[s] += -z / sg
                add(ssg, np.sum(z * z - 1.0) / sg)
            elif d == "cauchy":  # continuous.py:2287-2288
                a, sa = self._par(p.params[0], x)
                b, sb = self._par(p.params[1], x)
                u = xv - a
                den = b * b + u * u
                lp += np.sum(-np.log1p((u / b) ** 2)) - m * (np.log(np.pi) + np.log(b))
                gx[s] += -2.0 * u / den
                add(sa, np.sum(2.0 * u / den))
                add(sb, np.sum((u * u - b * b) / (b * den)))
            elif d == "halfcauchy":  # continuous.py:2383-2385 (+ Cauchy :2287-2288)
                b, sb = self._par(p.params[0], x)
                den = b * b + xv * xv
                lp += np.sum(-np.log1p((xv / b) ** 2)) + m * (np.log(2.0) - np.log(np.pi) - np.log(b))
                gx[s] += -2.0 * xv / den
                add(sb, np.sum((xv * xv - b * b) / (b * den)))
            elif d == "exponential":  # continuous.py:1478-1480 with mu = 1/lam
                lam, sl = self._par(p.params[0], x)
                lp += m * np.log(lam) - lam * np.sum(xv)
                gx[s] += -lam
                add(sl, m / lam - np.sum(xv))
            elif d == "studentt":  # continuous.py:1936-1944
                nu = float(p.params[0])
                mu, smu = self._par(p.params[1], x)
                sg, ssg = self._par(p.params[2], x)
                z = (xv - mu) / sg
                lp += m * (gammaln((nu + 1) / 2) - gammaln(nu / 2) - 0.5 * np.log(nu * np.pi) - np.log(sg)) \
                    - 0.5 * (nu + 1) * np.sum(np.log1p(z * z / nu))
                w = (nu + 1.0) * z / (sg * (nu + z * z))
                gx[s] += -w
                add(smu, np.sum(w))
                add(ssg, np.sum(-1.0 / sg + w * z))
            elif d == "uniform":  # continuous.py:309-314
                lo, hi = float(p.params[0]), float(p.params[1])
                lp += -m * np.log(hi - lo)
            elif d == "gamma":  # continuous.py:2512-2515
                al, be = float(p.params[0]), float(p.params[1])
                lp += m * (al * np.log(be) - gammaln(al)) + np.sum((al - 1.0) * np.log(xv) - be * xv)
                gx[s] += (al - 1.0) / xv - be
            elif d == "beta":  # continuous.py:1250-1256
                al, be = float(p.params[0]), float(p.params[1])
                lp += np.sum((al - 1.0) * np.log(xv) + (be - 1.0) * np.log1p(-xv)) \
                    - m * (gammaln(al) + gammaln(be) - gammaln(al + be))
                gx[s] += (al - 1.0) / xv - (be - 1.0) / (1.0 - xv)
            elif d == "lognormal":  # continuous.py:1807-1814
                mu, smu = self._par(p.params[0], x)
                sg, ssg = self._par(p.params[1], x)
                lx = np.log(xv)
                z = (lx - mu) / sg
                lp += np.sum(-0.5 * z * z - lx) - m * (HALF_LOG_2PI + np.log(sg))
                gx[s] += (-z / sg - 1.0) / xv
                add(smu, np.sum(z) / sg)
                add(ssg, np.sum(z * z - 1.0) / sg)
            else:  # pragma: no cover
                raise NotImplementedError(d)

        # ---- likelihoods -------------------------------------------------------------------------------------------
        for L in ir.likelihoods:
            y = np.asarray(L.y, dtype=np.float64)
            N = len(y)
            eta = np.zeros(N)
            fvals = []
            for t in L.terms:
                coef = np.ones(N) if t.coef is None else np.broadcast_to(np.asarray(t.coef, dtype=np.float64), (N,))
                vals = []
                for vn, idx in t.factors:
                    s = self._sl(vn)
                    xv = x[s]
                    vals.append(np.broadcast_to(xv, (N,)) if (idx is None and xv.size == 1) else (xv if idx is None else xv[idx]))
                fvals.append((coef, vals))
                eta += coef * np.prod(vals, axis=0)
            if L.dist == "normal":  # continuous.py:526-527
                if isinstance(L.sigma, Ref):
                    sg, ssg = self._par(L.sigma, x)
                else:
                    sg, ssg = np.asarray(L.sigma, dtype=np.float64), None
                z = (y - eta) / sg
                lp += np.sum(-0.5 * z * z - HALF_LOG_2PI - np.log(sg) * np.ones(N))
                r = z / sg
                add(ssg, np.sum((z * z - 1.0) / sg))
            elif L.dist == "bernoulli_logit":  # discrete.py:362-367 through PyTensor's stabilised log-sigmoid forms
                lp += np.sum(y * eta - _softplus(eta))
                r = y - _sigmoid(eta)
            elif L.dist == "poisson_log":  # discrete.py:581-586
                mu = np.exp(eta)
                lp += np.sum(y * eta - mu - gammaln(y + 1.0))
                r = y - mu
            elif L.dist == "studentt":  # continuous.py:1936-1944
                nu = float(L.nu)
                if isinstance(L.sigma, Ref):
                    sg, ssg = self._par(L.sigma, x)
                else:
                    sg, ssg = np.asarray(L.sigma, dtype=np.float64), None
                z = (y - eta) / sg
                lp += np.sum(gammaln((nu + 1) / 2) - gammaln(nu / 2) - 0.5 * np.log(nu * np.pi) - np.log(sg) * np.ones(N)
                             - 0.5 * (nu + 1) * np.log1p(z * z / nu))
                r = (nu + 1.0) * z / (sg * (nu + z * z))
                add(ssg, np.sum(-1.0 / sg + r * z))
            elif L.dist == "normal_logvar":  # Normal(0, exp(eta/2)), continuous.py:526-527
                w = y * y * np.exp(-eta)
                lp += np.sum(-0.5 * w - HALF_LOG_2PI - 0.5 * eta)
                r = 0.5 * w - 0.5
            else:  # pragma: no cover
                raise NotImplementedError(L.dist)
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

        # ---- AR(1) (timeseries.py:646-676 with ar_order 1, no constant term, init_dist = Normal(0, init_sigma)) -----
        for a in ir.ar1:
            s = self._sl(a.var)
            h = x[s]
            T = h.size
            phi, sphi = self._par(a.phi, x)
            sg, ssg = self._par(a.sigma, x)
            e = h[1:] - phi * h[:-1]
            i2 = 1.0 / (sg * sg)
            lp += -0.5 * (h[0] / a.init_sigma) ** 2 - HALF_LOG_2PI - np.log(a.init_sigma)
            lp += -0.5 * np.sum(e * e) * i2 - (T - 1) * (HALF_LOG_2PI + np.log(sg))
            g = np.zeros(T)
            g[0] -= h[0] / a.init_sigma**2
            g[1:] -= e * i2
            g[:-1] += phi * e * i2
            gx[s] += g
            add(sphi, np.sum(e * h[:-1]) * i2)
            add(ssg, (np.sum(e * e) * i2 - (T - 1)) / sg)

        return float(lp), gx * dxdq + djdq


def make_logp(ir: ModelIR) -> IrLogp:
    return IrLogp(ir)
