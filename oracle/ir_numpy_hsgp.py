"""TEST INFRASTRUCTURE ONLY -- NumPy evaluation q -> (logp, dlogp) of a ``pymc_b200.ir.ModelIR`` with spectral (HSGP) terms
and InverseGamma priors.

Layered like oracle/ir_numpy_beta.py: the rest of the model is evaluated by the oracle it is given (by default
ir_numpy_beta.make_logp, which covers every other factor of the closed set).  Each design term X x and each spectral term
f = Phi (z * s(theta)) is handed to that oracle as an elementwise offset u = X b of the predictor's length, a variable of its
own with no prior and no transform (b = x, or b = s(theta) * z).  The base oracle's gradient in u is d logp / d eta = r, so
g_b = X^T r, and this module takes it back to x, or to z, the amplitude a and the lengthscales l analytically, with
w_k = z_k s_k g_b_k:

  d/dz_k = s_k g_b_k,   d/da = sum_k w_k / a,   d/dl_d = sum_k w_k (1 / (2 l_d) + l_d omega_kd^2 h'(Q_k))

where log s_k = log a + (log C_D + sum_d log l_d + h(Q_k)) / 2 (``pymc_b200.ir.spectral_log_scale``).  InverseGamma(alpha,
beta) priors (continuous.py:2631-2640) add alpha log beta - lgamma(alpha) - (alpha + 1) log x - beta / x per element.

Pinned by tests/test_ir_hsgp.py against a 40-digit mpmath reference and central differences.  Only tests/ may import it.
"""
from __future__ import annotations

import copy

import numpy as np
from scipy.special import gammaln

from oracle import ir_numpy_beta, ir_numpy_ordinal
from pymc_b200.ir import Linear, ModelIR, Ref, Term, Var, is_design, spectral_log_const, spectral_log_scale


class HsgpLogp:
    def __init__(self, ir: ModelIR, base=None):
        ir.validate()
        self.ir, self.n, self.off = ir, ir.n, ir.offsets()
        ext = copy.deepcopy(ir)
        self.design = []  # (design or spectral term, the slice of its offset u in the extended q)
        n_ext = ir.n

        def swap(terms):
            nonlocal n_ext
            out = []
            for t in terms:
                if not is_design(t):
                    out.append(t)
                    continue
                N = np.shape(t.coef)[0]
                name = f"__design_u{len(self.design)}"
                ext.vars.append(Var(name, name, N))
                self.design.append((t, slice(n_ext, n_ext + N)))
                n_ext += N
                out.append(Term([(name, None)]))
            return out

        for L in ext.likelihoods:
            L.terms = swap(L.terms)
            if isinstance(L.psi, Linear):
                L.psi = Linear(swap(L.psi.terms))
        for p in ext.priors:
            p.params = tuple(Linear(swap(a.terms)) if isinstance(a, Linear) else a for a in p.params)
        self.invgamma = [p for p in ir.priors if p.dist == "inversegamma"]
        ext.priors = [p for p in ext.priors if p.dist != "inversegamma"]
        ext.deterministics = []
        self.n_ext = n_ext
        self.base = (base or ir_numpy_beta.make_logp)(ext)

    def _sl(self, name):
        v = self.ir.var(name)
        o = self.off[v.name]
        return slice(o, o + v.size)

    def constrained(self, q):
        return ir_numpy_ordinal.OrdinalLogp.constrained(self, q)

    def hyper(self, t, x):
        """(l [D], its slice in x or None, a, its slot in x or None) of spectral term t."""
        sp = t.spectral
        D = np.shape(sp.omega)[1]
        if isinstance(sp.ls, Ref):
            sl = self._sl(sp.ls.var)
            ls = np.broadcast_to(x[sl], (D,)).copy()
        else:
            sl, ls = None, np.broadcast_to(np.asarray(sp.ls, dtype=np.float64).reshape(-1), (D,)).copy()
        if isinstance(sp.amplitude, Ref):
            ao = self.off[self.ir.var(sp.amplitude.var).name]
            return ls, sl, x[ao], ao
        return ls, sl, float(sp.amplitude), None

    def scales(self, t, x):
        ls, _, a, _ = self.hyper(t, x)
        return np.exp(spectral_log_scale(t.spectral.cov, t.spectral.omega, ls, a))

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        x, dxdq = self.constrained(q)
        qe, parts = self.extended(x, q)
        lp, ge = self.base(qe)
        ge = np.asarray(ge, dtype=np.float64)
        g, gx = ge[: self.n].copy(), np.zeros(self.n)
        for (t, us), (s, z) in zip(self.design, parts):
            gb = np.asarray(t.coef, dtype=np.float64).T @ ge[us]
            zs = self._sl(t.factors[0][0])
            if s is None:
                gx[zs] += gb
                continue
            sp = t.spectral
            gx[zs] += s * gb
            w = z * s * gb
            ls, lsl, a, ao = self.hyper(t, x)
            if ao is not None:
                gx[ao] += np.sum(w) / a
            if lsl is not None:
                om2 = np.asarray(sp.omega, dtype=np.float64) ** 2
                Q = om2 @ (ls * ls)
                _, nu, c = spectral_log_const(sp.cov, len(ls))
                dh = np.full_like(Q, -0.5) if sp.cov == "expquad" else -nu / (c + Q)
                dl = np.sum(w) / (2.0 * ls) + ls * ((w * dh) @ om2)
                if lsl.stop - lsl.start == 1:
                    gx[lsl] += np.sum(dl)
                else:
                    gx[lsl] += dl
        for p in self.invgamma:
            al, be = (float(a) for a in p.params)
            sl = self._sl(p.var)
            xv = x[sl]
            lp += float(np.sum(al * np.log(be) - gammaln(al) - (al + 1.0) * np.log(xv) - be / xv))
            gx[sl] += -(al + 1.0) / xv + be / xv**2
        return float(lp), g + gx * dxdq

    def extended(self, x, q):
        """(q with every offset u = X b filled in, [(s or None, b)] per design / spectral term)."""
        qe = np.concatenate([q, np.zeros(self.n_ext - self.n)])
        parts = []
        for t, us in self.design:
            b = x[self._sl(t.factors[0][0])]
            s = self.scales(t, x) if t.spectral is not None else None
            qe[us] = np.asarray(t.coef, dtype=np.float64) @ (b if s is None else s * b)
            parts.append((s, b))
        return qe, parts


def make_logp(ir: ModelIR, base=None):
    """ir_numpy_beta.make_logp (or ``base``) for any model of the closed set, with spectral terms and InverseGamma priors."""
    has_spec = any(t.spectral is not None for L in ir.likelihoods for t in L.terms + (L.psi.terms if isinstance(L.psi, Linear) else [])) \
        or any(t.spectral is not None for p in ir.priors for a in p.params if isinstance(a, Linear) for t in a.terms)
    if has_spec or any(p.dist == "inversegamma" for p in ir.priors):
        return HsgpLogp(ir, base)
    return (base or ir_numpy_beta.make_logp)(ir)
