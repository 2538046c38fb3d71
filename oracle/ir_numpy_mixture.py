"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` with simplex variables,
Dirichlet priors and finite mixtures (``MIXTURE_LIKS``).

Layered like oracle/ir_numpy_survival.py: the rest of the model (every other factor, the priors of the components and
sigma, every other transform) is evaluated by the oracle it is given (by default ir_numpy_survival.make_logp, which covers
every other factor of the closed set).  This module adds, with every constant:

  simplex        SimplexTransform (transforms.py:1091-1116): w = softmax([z, -sum z]), log w_k = z_k - lse(z) (finite where
                 w_k underflows); log|J| = log K + sum_k log w_k, the reference's log_jac_det
  dirichlet      Dirichlet(a) (multivariate.py:557-585): lgamma(sum a) - sum lgamma(a_k) + sum (a_k - 1) log w_k
  mixtures       mixture_logprob (mixture.py:469-494): log p(y_i) = logsumexp_k(log w_k + log f_k(y_i)) with
                 f_k = Normal(eta_i + mu_k, sigma_k) or Poisson(lam_k e^eta_i)

The gradient reaches the simplex through G_k = d logp / d log w_k and d/dz_j = (G_j - w_j S) - (G_K - w_K S), S = sum G.
Pinned by tests/test_ir_mixture.py against a 40-digit mpmath reference (itself checked against scipy.stats) and central
differences.  Only tests/ may import it.
"""
from __future__ import annotations

import dataclasses

import numpy as np
from scipy.special import gammaln, logsumexp

from oracle import ir_numpy_bounded, ir_numpy_ordinal, ir_numpy_survival, ir_numpy_zero_inflated
from pymc_b200.ir import MIXTURE_LIKS, ORDERED_TRANSFORMS, ModelIR, Ref

HALF_LOG_2PI = 0.5 * np.log(2.0 * np.pi)


def simplex_log_weights(z):
    """log w_k = z~_k - lse(z~), z~ = [z, -sum z], along the last axis."""
    z = np.asarray(z, dtype=np.float64)
    ze = np.concatenate([z, -np.sum(z, axis=-1, keepdims=True)], axis=-1)
    return ze - logsumexp(ze, axis=-1, keepdims=True)


def mixture_terms(dist, y, eta, lw, c, s):
    """(log p_i with every constant, d / d eta_i, rho [N, K], d log f / d c_k [N, K], d log f / d sigma_k [N, K]) of every
    observation: lw the K log weights, c the components mu_k or lam_k, s the K sigma_k (Normal)."""
    y, eta = np.asarray(y, dtype=np.float64)[:, None], np.asarray(eta, dtype=np.float64)[:, None]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):  # lam e^eta may overflow: f_k = 0
        if dist == "normal_mixture":
            z = (y - eta - c) / s
            lf = -0.5 * z * z - np.log(s) - HALF_LOG_2PI
            de, dc, ds = z / s, z / s, (z * z - 1.0) / s
        else:
            mu = c * np.exp(eta)
            lf = y * (np.log(c) + eta) - mu - gammaln(y + 1.0)
            de, dc, ds = y - mu, (y - mu) / c, np.zeros_like(mu)
        l = lw + lf
        lse = logsumexp(l, axis=1)
        drop = np.isneginf(l)  # a weight of 0, or a density that underflows to 0: no responsibility, no derivative
        rho = np.where(drop, 0.0, np.exp(l - lse[:, None]))
        de, dc, ds = (np.where(drop, 0.0, d) for d in (de, dc, ds))
    return lse, np.sum(rho * de, axis=1), rho, dc, ds


class MixtureLogp:
    def __init__(self, ir: ModelIR, base=None):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()
        self.mix = [L for L in ir.likelihoods if L.dist in MIXTURE_LIKS]
        self.simplex = [v for v in ir.vars if v.transform == "simplex"]
        self.dirichlet = [p for p in ir.priors if p.dist == "dirichlet"]
        self.ordered = [v for v in ir.vars if v.transform in ORDERED_TRANSFORMS]
        # the base sees each simplex variable as an unused untransformed one: it adds nothing there
        rest = dataclasses.replace(
            ir, vars=[dataclasses.replace(v, transform=None) if v.transform == "simplex" else v for v in ir.vars],
            priors=[p for p in ir.priors if p.dist != "dirichlet"],
            likelihoods=[L for L in ir.likelihoods if L.dist not in MIXTURE_LIKS])
        self.base = (base or ir_numpy_survival.make_logp)(rest)

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def constrained(self, q):
        return ir_numpy_ordinal.OrdinalLogp.constrained(self, q)

    def eta(self, L, x):
        return ir_numpy_bounded.BoundedLogp.eta(self, L, x)

    def log_weights(self, q):
        """simplex variable name -> its K log weights."""
        return {v.name: simplex_log_weights(q[self._sl(v.name)]) for v in self.simplex}

    def blocks(self, L, x, lws):
        """(log w, components, sigma (K values or None)) of mixture L."""
        K = L.n_components(self.ir)
        if isinstance(L.weights, Ref):
            lw = lws[self.ir.var(L.weights.var).name]
        else:
            with np.errstate(divide="ignore"):
                lw = np.log(np.asarray(L.weights, dtype=np.float64))
        c = x[self._sl(L.components.var)] if isinstance(L.components, Ref) else np.asarray(L.components, dtype=np.float64)
        s = None
        if L.dist == "normal_mixture":
            s = x[self._sl(L.sigma.var)] if isinstance(L.sigma, Ref) else np.asarray(L.sigma, dtype=np.float64)
            s = np.broadcast_to(s, (K,))
        return lw, c, s

    def loglik(self, L, x, q):
        """log p(y_i | x) of every observation of mixture L, with every constant."""
        lw, c, s = self.blocks(L, x, self.log_weights(np.asarray(q, dtype=np.float64)))
        return mixture_terms(L.dist, L.y, self.eta(L, x)[0], lw, c, s)[0]

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        lp, g = self.base(q)
        g = np.array(g, dtype=np.float64)
        x, dxdq = self.constrained(q)
        lws = self.log_weights(q)
        G = {name: np.ones(len(lw)) for name, lw in lws.items()}  # d log|J| / d log w_k = 1
        for name, lw in lws.items():
            lp += float(np.log(len(lw)) + np.sum(lw))
        for p in self.dirichlet:
            name = self.ir.var(p.var).name
            a = np.broadcast_to(np.asarray(p.params[0], dtype=np.float64), lws[name].shape)
            lp += float(gammaln(np.sum(a)) - np.sum(gammaln(a)) + np.sum((a - 1.0) * lws[name]))
            G[name] = G[name] + (a - 1.0)
        gx = np.zeros(self.n)
        for L in self.mix:
            eta, parts = self.eta(L, x)
            lw, c, s = self.blocks(L, x, lws)
            lpi, r, rho, dc, ds = mixture_terms(L.dist, L.y, eta, lw, c, s)
            lp += float(np.sum(lpi))
            ir_numpy_zero_inflated.ZeroInflatedLogp._pull(self, gx, parts, r)
            if isinstance(L.weights, Ref):
                name = self.ir.var(L.weights.var).name
                G[name] = G[name] + rho.sum(axis=0)
            if isinstance(L.components, Ref):
                gx[self._sl(L.components.var)] += np.sum(rho * dc, axis=0)
            if isinstance(L.sigma, Ref):
                sl = self._sl(L.sigma.var)
                gs = np.sum(rho * ds, axis=0)
                gx[sl] += gs if sl.stop - sl.start > 1 else gs.sum()
        out = g + gx * dxdq
        for v in self.ordered:  # the chain rule of what this layer added, through the cumulative sum
            sl = self._sl(v.name)
            S = np.cumsum(gx[sl][::-1])[::-1]
            add = np.exp(q[sl]) * S
            if v.transform == "ordered":
                add[0] = S[0]
            out[sl] = g[sl] + add
        for v in self.simplex:
            sl = self._sl(v.name)
            Gv, w = G[v.name], np.exp(lws[v.name])
            S = np.sum(Gv)
            out[sl] = (Gv[:-1] - w[:-1] * S) - (Gv[-1] - w[-1] * S)
        return float(lp), out


def make_logp(ir: ModelIR, base=None):
    """ir_numpy_survival.make_logp (or ``base``) for any model of the closed set, with simplex variables, Dirichlet priors
    and mixtures."""
    if any(L.dist in MIXTURE_LIKS for L in ir.likelihoods) or any(v.transform == "simplex" for v in ir.vars):
        return MixtureLogp(ir, base)
    return (base or ir_numpy_survival.make_logp)(ir)
