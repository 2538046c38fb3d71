"""Survival likelihoods of the model IR (``ir.SURVIVAL_LIKS``): the Weibull with a log link (the Exponential is its alpha =
1) and the LogNormal, plain, censored or truncated.

``_mp_logp`` writes the joint log-density with mpmath at 40 digits from the published definitions: the Weibull's
log f, log S = -t and log F = log(1 - e^-t), its truncated normaliser log(e^{-tA} - e^{-tB}), and the LogNormal as the
Normal of log y minus log y, with Phi through erfc in both tails; the gradient is ``mpmath.diff``.  It reads the ``ModelIR``
dataclasses and nothing else of the package or of oracle/.  S = sum |additive pieces|: logp is compared to 1e-13 S; the
gradient to 1e-12 max(1, |g|_inf) plus 1e-15 G, G the sum of the sizes of the parts d logp / d eta and d logp / d alpha or
sigma are formed from (``_mp_grad_pieces``), as in tests/test_ir_bounded.py.

CPU: the reference against scipy.stats, the oracle (oracle/ir_numpy_survival.py) against the reference and central
differences on every catalogue case, the support rule through validate() and the C ABI, the lowered tables, ``specialise``
/ ``fuse_design_columns``, and the sampler's data groups through the oracle-backed stand-in.  GPU: the generic device
function against both, the pointwise log-likelihood, fixed-step, lock-step and adaptive NUTS against the oracle sampler."""
import ctypes
import zlib
from functools import lru_cache

import mpmath
import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import stats
from b200_helpers import (adaptive_against_oracle, fd_grad, fixed_step_against_oracle, logp_at_both_team_shapes,
                          random_dense_cov, refusal_after_edit)
from test_ir_bounded import _mp_constrain, _mp_eta, _mp_Phi, _mp_Q, _mp_side, assert_close_to_reference
from test_ir_closed_set import MP_DPS

from pymc_b200 import _lib, ir
from pymc_b200.ir import Likelihood, ModelIR, Prior, Ref, Term, Var


# ------------------------------------------------------------------------------------------------------------------------
# the high-precision reference
# ------------------------------------------------------------------------------------------------------------------------
def _mp_log1mexp(t):
    """log(1 - e^-t) at the working precision (40 digits keep ~28 of them at t = 1e-12)."""
    return mp.log(-mp.expm1(-t))


def _mp_lik_pieces(dist, y, eta, p, lo, hi):
    """Pieces of log p(y | eta) of one survival observation; p is alpha (Weibull) or sigma (LogNormal); lo / hi are mpf
    or +-mp.inf, a lower bound <= 0 being open."""
    cens, trunc = dist.startswith("censored"), dist.startswith("truncated")
    lo = lo if lo > 0 else mpf(0)
    if dist in ir.WEIBULL_LIKS:
        t_of = lambda v: mp.exp(p * (mp.log(v) - eta))  # noqa: E731
        u = mp.log(y) - eta
        if cens and y == hi:
            return [-t_of(y)]
        if cens and y == lo:
            return [_mp_log1mexp(t_of(y))]
        out = [mp.log(p), -eta, (p - 1) * u, -t_of(y)]
        if trunc:
            sa = mp.exp(-t_of(lo)) if lo > 0 else mpf(1)
            sb = mp.exp(-t_of(hi)) if hi != mp.inf else mpf(0)
            out.append(-mp.log(sa - sb))
        return out
    ly = mp.log(y)
    z = (ly - eta) / p
    if cens and y == hi:
        return [mp.log(_mp_Q(z))]
    if cens and y == lo:
        return [mp.log(_mp_Phi(z))]
    out = [-z * z / 2, -mp.log(p), -mp.log(2 * mp.pi) / 2, -ly]
    if trunc:
        a = (mp.log(lo) - eta) / p if lo > 0 else -mp.inf
        b = (mp.log(hi) - eta) / p if hi != mp.inf else mp.inf
        out.append(-mp.log(_mp_Q(a) - _mp_Q(b) if a >= 0 else _mp_Phi(b) - _mp_Phi(a)))
    return out


def _mp_par(m, L, x):
    """alpha or sigma of every observation."""
    N = len(L.y)
    p = L.alpha if L.dist in ir.WEIBULL_LIKS else L.sigma
    if isinstance(p, Ref):
        return [x[m.var(p.var).name][0]] * N
    return [mpf(float(v)) for v in np.broadcast_to(p, (N,))]


def _mp_prior(p, x, vn, par):
    a = [par(t, x) for t in p.params]
    if p.dist == "normal":
        return [t for xi in x[vn] for t in (-((xi - a[0]) / a[1]) ** 2 / 2, -mp.log(a[1]), -mp.log(2 * mp.pi) / 2)]
    if p.dist == "halfnormal":
        return [t for xi in x[vn] for t in (-(xi / a[0]) ** 2 / 2, -mp.log(a[0]), mp.log(2) / 2 - mp.log(mp.pi) / 2)]
    assert p.dist == "uniform"
    return [-mp.log(a[1] - a[0]) for _ in x[vn]]


def _mp_factors(m):
    name = lambda r: m.var(r).name  # noqa: E731
    par = lambda a, x: x[name(a.var)][0] if isinstance(a, Ref) else mpf(float(a))  # noqa: E731
    out = []
    for p in m.priors:
        vn = name(p.var)
        out.append(({vn} | {name(a.var) for a in p.params if isinstance(a, Ref)},
                    lambda x, p=p, vn=vn: _mp_prior(p, x, vn, par)))
    for L in m.likelihoods:
        N = len(L.y)
        y = [mpf(float(v)) for v in L.y]
        lo_, hi_ = L.bounds()
        lo, hi = [_mp_side(v) for v in lo_], [_mp_side(v) for v in hi_]
        deps = {name(vn) for t in L.terms for vn, _ in t.factors}
        slot = L.alpha if L.dist in ir.WEIBULL_LIKS else L.sigma
        if isinstance(slot, Ref):
            deps.add(name(slot.var))

        def lik(x, L=L, y=y, lo=lo, hi=hi, N=N):
            eta, p = _mp_eta(m, L, x), _mp_par(m, L, x)
            return [t for i in range(N) for t in _mp_lik_pieces(L.dist, y[i], eta[i], p[i], lo[i], hi[i])]
        out.append((deps, lik))
    return out


def _mp_logp(m, q):
    with mp.workdps(MP_DPS):
        x, jac = _mp_constrain(m, [mpf(float(t)) for t in q])
        pieces = [t for j in jac for t in j] + [t for _, f in _mp_factors(m) for t in f(x)]
        return float(mp.fsum(pieces)), float(mp.fsum(abs(t) for t in pieces))


def _mp_grad(m, q):
    facs, off, g = _mp_factors(m), m.offsets(), np.empty(m.n)
    with mp.workdps(MP_DPS):
        q0 = [mpf(float(t)) for t in q]
        for v in m.vars:
            fs = [f for deps, f in facs if v.name in deps]
            for j in range(off[v.name], off[v.name] + v.size):
                def h(t, j=j, fs=fs):
                    qq = q0[:]
                    qq[j] = t
                    x, jac = _mp_constrain(m, qq)
                    return mp.fsum(jac[j] + [p for f in fs for p in f(x)])
                g[j] = float(mpmath.diff(h, q0[j]))
    return g


def _mp_grad_pieces(m, q):
    """G = the sum over observations of the sizes of the parts d logp / d eta and d logp / d alpha or sigma are formed
    from.  Weibull: (1 + alpha + |u|) (1 + t(y) + t(A) + t(B)) at each bound present, so a narrow window far in the tail,
    whose parts of size alpha t cancel to O(1), carries rounding of 1e-16 G.  LogNormal: tests/test_ir_bounded.py's G on
    log y and log bounds."""
    with mp.workdps(MP_DPS):
        x, _ = _mp_constrain(m, [mpf(float(t)) for t in q])
        G = mpf(0)
        for L in m.likelihoods:
            eta, par = _mp_eta(m, L, x), _mp_par(m, L, x)
            lo_, hi_ = L.bounds()
            for i in range(len(L.y)):
                y, p, lo, hi = mpf(float(L.y[i])), par[i], _mp_side(lo_[i]), _mp_side(hi_[i])
                lo = lo if lo > 0 else mpf(0)
                if L.dist in ir.WEIBULL_LIKS:
                    u = mp.log(y) - eta[i]
                    ts = mp.exp(p * u) + sum(mp.exp(p * (mp.log(b) - eta[i])) for b in (lo, hi) if 0 < b < mp.inf)
                    G += (1 + p + abs(u)) * (1 + ts)
                    continue
                z = (mp.log(y) - eta[i]) / p
                G += (1 + abs(z)) * (1 + abs(z)) / p
                if L.dist == "censored_lognormal" and (y == lo or y == hi):
                    zc = z if y == lo else -z
                    G += mp.npdf(zc) / _mp_Phi(zc) * (1 + abs(zc)) / p
                elif L.dist == "truncated_lognormal":
                    a = (mp.log(lo) - eta[i]) / p if lo > 0 else -mp.inf
                    b = (mp.log(hi) - eta[i]) / p if hi != mp.inf else mp.inf
                    Z = _mp_Q(a) - _mp_Q(b) if a >= 0 else _mp_Phi(b) - _mp_Phi(a)
                    G += sum(mp.npdf(c) * (1 + abs(c)) for c in (a, b) if abs(c) != mp.inf) / (p * Z)
        return float(G)


# ------------------------------------------------------------------------------------------------------------------------
# the case catalogue
# ------------------------------------------------------------------------------------------------------------------------
PARAMS = {"const": lambda N, rng, d: 1.7 if d in ir.WEIBULL_LIKS else 0.8,
          "ref_log": lambda N, rng, d: Ref("p_log__"), "ref_int": lambda N, rng, d: Ref("p_interval__"),
          "obs": lambda N, rng, d: rng.uniform(0.5, 1.5, N)}


def _param_vars(kind):
    if kind == "ref_log":
        return [Var("p_log__", "p", 1, "log")], [Prior("halfnormal", "p_log__", (2.0,))]
    if kind == "ref_int":
        return [Var("p_interval__", "p", 1, "interval", (0.3, 12.0))], [Prior("uniform", "p_interval__", (0.3, 12.0))]
    return [], []


def _regression_case(dist, kind, shape, rng, N=12):
    """b0 + b1 x (or a design term and a group effect) under a survival likelihood with bounds of the given shape."""
    x = rng.standard_normal(N)
    eta = 0.3 + 0.5 * x
    y = np.exp(eta) * (rng.weibull(1.5, N) if dist in ir.WEIBULL_LIKS else np.exp(0.8 * rng.standard_normal(N)))
    vars_ = [Var("b0", "b0", 1), Var("b1", "b1", 1)]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "b1", (0.0, 1.0))]
    terms = [Term([("b0", None)]), Term([("b1", None)], coef=x)]
    if shape == "design":
        X = np.column_stack([np.ones(N), x, rng.standard_normal(N)])
        vars_ = [Var("beta", "beta", 3), Var("g", "g", 3)]
        priors = [Prior("normal", "beta", (0.0, 1.5)), Prior("normal", "g", (0.0, 1.0))]
        terms = [Term([("beta", None)], coef=X), Term([("g", np.arange(N, dtype=np.int32) % 3)])]
    pv, pp = _param_vars(kind)
    vars_, priors = vars_ + pv, priors + pp
    lower = upper = None
    q = np.sort(y)
    if dist.startswith("censored"):
        if shape == "lower":  # left-censored at one detection limit
            lower = float(q[3])
        elif shape == "upper":  # right-censored at each observation's follow-up time
            upper = np.where(rng.random(N) < 0.5, y * rng.uniform(0.4, 1.0, N), np.inf)
        elif shape in ("both", "design"):
            lower, upper = float(q[2]), float(q[-3])
        else:  # "mixed": per-observation bounds, open sides written as 0, -inf and +inf
            lower = np.where(rng.random(N) < 0.5, y * rng.uniform(0.3, 1.0, N), np.where(rng.random(N) < 0.5, 0.0, -np.inf))
            upper = np.where(rng.random(N) < 0.5, y * rng.uniform(1.0, 3.0, N), np.inf)
            k = rng.choice(N, 4, replace=False)
            lower[k[:2]], upper[k[2:]] = y[k[:2]], y[k[2:]]  # some exactly at a bound of their own
        lo = np.broadcast_to(-np.inf if lower is None else lower, (N,))
        hi = np.broadcast_to(np.inf if upper is None else upper, (N,))
        y = np.clip(y, lo, hi)
    elif dist.startswith("truncated"):
        if shape == "lower":  # delayed entry, none for some subjects
            lower = np.where(rng.random(N) < 0.3, 0.0, y * rng.uniform(0.2, 0.95, N))
        elif shape == "upper":
            upper = float(q[-1] * 1.2)
        else:  # "two" / "design": windows around y, two of them with t(B) - t(A) ~ 1e-6
            lower, upper = y * rng.uniform(0.3, 0.9, N), y * rng.uniform(1.1, 2.5, N)
            lower[:2], upper[:2] = y[:2] * (1 - 3e-7), y[:2] * (1 + 3e-7)
            if dist == "truncated_lognormal":  # a window 1e-3 wide in log y: log bounds lose digits below it
                lower[:2], upper[:2] = y[:2] * (1 - 5e-4), y[:2] * (1 + 5e-4)
    L = Likelihood(dist, y, terms, lower=lower, upper=upper,
                   **({"alpha": PARAMS[kind](N, rng, dist)} if dist in ir.WEIBULL_LIKS else {"sigma": PARAMS[kind](N, rng, dist)}))
    return ModelIR(vars=vars_, priors=priors, likelihoods=[L])


def _weibull_tail_case(dist, alpha):
    """eta = b0 with b0 = 0 at the first point: censored, t(y) from 1e-12 (left) to 700 (right); truncated, windows with
    t(B) - t(A) ~ 1e-6 at t ~ 1 and ~ 300 and a delayed entry at t(A) = 700."""
    r = lambda t: float(t ** (1.0 / alpha))  # noqa: E731  (the y of a given t at eta = 0)
    if dist == "censored_weibull_log":
        t = np.array([1e-12, 1e-6, 0.01, 0.5, 3.0, 50.0, 300.0, 700.0, 1.0, 2.0])
        y = np.array([r(v) for v in t])
        lower = np.where(np.arange(10) < 4, y, 0.0)
        upper = np.where((np.arange(10) >= 4) & (np.arange(10) < 8), y, np.inf)
    else:
        ta = np.array([1.0, 300.0, 700.0, 0.2, 1e-10, 40.0])
        lower = np.array([r(v) for v in ta])
        upper = np.array([r(1.0 + 1e-6), r(300.0 + 1e-6), np.inf, r(0.3), r(2.0), r(40.5)])
        y = np.where(np.isfinite(upper), lower + 0.5 * (np.where(np.isfinite(upper), upper, 0.0) - lower), lower * 1.01)
        lower[4] = 0.0  # an open lower side with only an upper bound
        y[4] = r(1.0)
    return ModelIR(vars=[Var("b0", "b0", 1)], priors=[Prior("normal", "b0", (0.0, 3.0))],
                   likelihoods=[Likelihood(dist, y, [Term([("b0", None)])], alpha=alpha, lower=lower, upper=upper)])


def _lognormal_tail_case(dist):
    """eta = b0, sigma = 1 in log y: censoring points at log y from -30 to 30, truncated windows 1e-3 wide in a tail."""
    if dist == "censored_lognormal":
        ly = np.array([-30.0, -8.0, -1.5, 0.2, 1.2, 8.0, 30.0, 0.0])
        y = np.exp(ly)
        lower = np.where(np.arange(8) < 3, y, 0.0)
        upper = np.where((np.arange(8) >= 3) & (np.arange(8) < 7), y, np.inf)
    else:
        la = np.array([-20.0, -3.0, 0.5, 19.0, 29.999, -0.0005])
        lb = np.array([-19.99, -2.0, 0.501, 20.0, 30.0, 0.0005])
        lower, upper = np.exp(la), np.exp(lb)
        y = np.exp(0.5 * (la + lb))
    return ModelIR(vars=[Var("b0", "b0", 1)], priors=[Prior("normal", "b0", (0.0, 3.0))],
                   likelihoods=[Likelihood(dist, y, [Term([("b0", None)])], sigma=1.0, lower=lower, upper=upper)])


CASES = {}
for _d in ir.SURVIVAL_LIKS:
    _w = _d in ir.WEIBULL_LIKS
    _kinds = ("const", "ref_log", "ref_int") if _w else ("const", "ref_log", "obs")
    _shapes = {"censored": ("lower", "upper", "both", "mixed", "design"), "truncated": ("lower", "upper", "two", "design")}.get(
        _d.split("_")[0], ("plain", "design", "again"))
    for _j, _sh in enumerate(_shapes):
        _k = _kinds[_j % 3]
        CASES[f"{_d}-{_sh}-{_k}"] = (lambda rng, d=_d, k=_k, sh=_sh: _regression_case(d, k, sh, rng))
    if _d.startswith(("censored", "truncated")):
        if _w:
            for _a in (0.3, 1.0, 12.0):
                CASES[f"{_d}-tails-alpha{_a:g}"] = (lambda rng, d=_d, a=_a: _weibull_tail_case(d, a))
        else:
            CASES[f"{_d}-tails"] = (lambda rng, d=_d: _lognormal_tail_case(d))
CASE_IDS = list(CASES)


def build(cid):
    return CASES[cid](np.random.default_rng(zlib.crc32(cid.encode())))


def points(m, cid):
    """The initial point + U(-1, 1) (twice; U(-0.3, 0.3) for the shape 12 regression cases); for the tail cases b0 in
    {0, -0.3, 0.3}, which moves every t by e^{-+0.3 alpha}."""
    rng = np.random.default_rng(zlib.crc32(cid.encode()) + 1)
    q0 = m.initial_point()
    if "tails" in cid:
        return np.array([[b] for b in (0.0, -0.3, 0.3)])
    return np.array([q0 + rng.uniform(-1.0, 1.0, m.n) for _ in range(2)])


@lru_cache(maxsize=None)
def mp_reference(cid):
    m = build(cid)
    Q = points(m, cid)
    lp, S = np.array([_mp_logp(m, q) for q in Q]).T
    return Q, lp, S, np.array([_mp_grad(m, q) for q in Q]), np.array([_mp_grad_pieces(m, q) for q in Q])


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference and the oracle
# ------------------------------------------------------------------------------------------------------------------------
def _mp_one(dist, y, eta, p, lo=-np.inf, hi=np.inf):
    with mp.workdps(MP_DPS):
        return float(mp.fsum(_mp_lik_pieces(dist, mpf(y), mpf(eta), mpf(p), _mp_side(lo), _mp_side(hi))))


def test_mp_pieces_equal_scipy():
    """The Weibull's logpdf / logsf / logcdf, the Exponential, the LogNormal's three and both truncated normalisers."""
    for y, eta, a in [(0.5, 0.0, 1.5), (3.0, 0.4, 0.3), (1e-3, -0.2, 12.0), (7.0, 1.0, 1.0), (2.0, 0.0, 4.0), (0.05, 0.3, 0.7)]:
        w = stats.weibull_min(a, scale=np.exp(eta))
        for lo, hi, want in ((-np.inf, np.inf, w.logpdf(y)), (-np.inf, y, w.logsf(y)), (y, np.inf, w.logcdf(y))):
            d = "weibull_log" if (lo, hi) == (-np.inf, np.inf) else "censored_weibull_log"
            got = _mp_one(d, y, eta, a, lo, hi)
            assert abs(got - want) <= 1e-12 * max(1.0, abs(want)), (y, eta, a, lo, hi, got, want)
        if a == 1.0:
            assert abs(_mp_one("weibull_log", y, eta, a) - stats.expon.logpdf(y, scale=np.exp(eta))) <= 1e-13
        for lo, hi in ((0.5 * y, 2.0 * y), (0.9 * y, np.inf), (0.0, 1.5 * y)):
            want = w.logpdf(y) - np.log(w.cdf(hi) - w.cdf(lo))
            got = _mp_one("truncated_weibull_log", y, eta, a, lo, hi)
            assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), (y, lo, hi, got, want)  # scipy: cdf(hi) - cdf(lo)
    for y, eta, s in [(0.5, 0.0, 1.0), (3.0, 0.4, 0.3), (1e-3, -0.2, 2.0), (40.0, 1.0, 0.7)]:
        ln = stats.lognorm(s, scale=np.exp(eta))
        for lo, hi, want in ((-np.inf, np.inf, ln.logpdf(y)), (-np.inf, y, ln.logsf(y)), (y, np.inf, ln.logcdf(y))):
            d = "lognormal" if (lo, hi) == (-np.inf, np.inf) else "censored_lognormal"
            got = _mp_one(d, y, eta, s, lo, hi)
            assert abs(got - want) <= 1e-12 * max(1.0, abs(want)), (y, eta, s, lo, hi, got, want)
        for lo, hi in ((0.5 * y, 2.0 * y), (0.9 * y, np.inf), (0.0, 1.5 * y)):
            want = ln.logpdf(y) - np.log(ln.cdf(hi) - ln.cdf(lo))
            got = _mp_one("truncated_lognormal", y, eta, s, lo, hi)
            assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), (y, lo, hi, got, want)  # scipy: cdf(hi) - cdf(lo)


def test_the_catalogue_covers_the_survival_forms():
    seen = set()
    for cid in CASE_IDS:
        m = build(cid)
        m.validate()
        L = m.likelihoods[0]
        lo, hi = L.bounds()
        p = L.alpha if L.dist in ir.WEIBULL_LIKS else L.sigma
        kind = ("ref_int" if m.var(p.var).transform == "interval" else "ref_log") if isinstance(p, Ref) else \
            ("obs" if np.ndim(p) == 1 else "const")
        seen |= {(L.dist, "any"), (L.dist, kind)}
        seen.add((L.dist, "design")) if any(ir.is_design(t) for t in L.terms) else None
        if L.dist.startswith("censored"):
            at_lo, at_hi = np.any(L.y == lo), np.any(L.y == hi)
            seen.add((L.dist, {(True, False): "lower", (False, True): "upper", (True, True): "both"}[(at_lo, at_hi)]))
            if np.ndim(L.lower) == 1 and np.any(L.lower == 0.0) and np.any(np.isneginf(L.lower)) and np.any(np.isinf(hi)):
                seen.add((L.dist, "mixed_open"))
        if L.dist.startswith("truncated"):
            has_lo, has_hi = np.any(lo > 0), np.any(np.isfinite(hi))
            seen.add((L.dist, {(True, False): "lower", (False, True): "upper", (True, True): "two"}[(has_lo, has_hi)]))
    for d in ir.SURVIVAL_LIKS:
        kinds = ("const", "ref_log", "ref_int") if d in ir.WEIBULL_LIKS else ("const", "ref_log", "obs")
        assert {(d, k) for k in kinds + ("design",)} <= seen, d
    for d in ("censored_weibull_log", "censored_lognormal"):
        assert {(d, s) for s in ("lower", "upper", "both", "mixed_open")} <= seen, d
    for d in ("truncated_weibull_log", "truncated_lognormal"):
        assert {(d, s) for s in ("lower", "upper", "two")} <= seen, d
    # the Weibull tails: t from 1e-12 (log F) to 700 (log S), windows with t(B) - t(A) ~ 1e-6, alpha from 0.3 to 12
    for a in (0.3, 1.0, 12.0):
        L = build(f"censored_weibull_log-tails-alpha{a:g}").likelihoods[0]
        t = L.y ** a
        assert np.isclose(t[L.y == L.bounds()[0]].min(), 1e-12) and np.isclose(t[L.y == L.bounds()[1]].max(), 700.0)
        L = build(f"truncated_weibull_log-tails-alpha{a:g}").likelihoods[0]
        lo, hi = L.bounds()
        two = (lo > 0) & np.isfinite(hi)
        assert np.min((hi ** a - lo ** a)[two]) < 2e-6
    alphas = {float(build(c).likelihoods[0].alpha) for c in CASE_IDS if "alpha" in c}
    assert min(alphas) == 0.3 and max(alphas) == 12.0


@pytest.mark.parametrize("cid", CASE_IDS)
def test_oracle_matches_the_mp_reference_and_central_differences(cid):
    from oracle import ir_numpy_survival

    m = build(cid)
    f = ir_numpy_survival.make_logp(m)
    Q, lp_mp, S, g_mp, G = mp_reference(cid)
    lp, g = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    assert np.all(np.isfinite(lp)) and np.all(np.isfinite(g)), cid
    assert_close_to_reference(lp, g, lp_mp, S, g_mp, G, cid)
    gf = fd_grad(f, Q[0], h=1e-6)
    assert np.max(np.abs(gf - g[0])) <= 1e-5 * max(1.0, np.max(np.abs(g[0]))), cid


def scipy_pointwise(L, eta, p):
    """log p(y_i | eta_i) of a survival likelihood from scipy.stats (a truncated one with its normaliser from sf)."""
    y = np.asarray(L.y, dtype=np.float64)
    lo, hi = L.bounds()
    d = stats.weibull_min(p, scale=np.exp(eta)) if L.dist in ir.WEIBULL_LIKS else stats.lognorm(p, scale=np.exp(eta))
    if L.dist.startswith("censored"):
        return np.where(y == lo, d.logcdf(y), np.where(y == hi, d.logsf(y), d.logpdf(y)))
    if L.dist.startswith("truncated"):
        return d.logpdf(y) - np.log(d.sf(np.where(lo > 0, lo, 0.0)) - d.sf(hi))
    return d.logpdf(y)


SCIPY_BUILDS = [("weibull", "right_censored"), ("exponential", "plain"), ("exponential", "right_censored"),
                ("lognormal", "entry_truncated"), ("weibull", "entry_truncated"), ("lognormal", "plain")]


def test_oracle_pointwise_equals_scipy_on_the_builders():
    from oracle import ir_numpy_survival

    for dist, observe in SCIPY_BUILDS:
        m = ir.survival_regression_ir(dist, observe, n_obs=80)
        f = ir_numpy_survival.make_logp(m)
        q = m.initial_point() + np.random.default_rng(2).uniform(-0.5, 0.5, m.n)
        x, _ = f.constrained(q)
        L = m.likelihoods[0]
        want = scipy_pointwise(L, f.eta(L, x)[0], f.param(L, x)[0])
        np.testing.assert_allclose(f.loglik(L, x), want, rtol=1e-11, atol=1e-11, err_msg=f"{dist} {observe}")
        if dist == "exponential" and observe == "plain":  # pm.Exponential.logp = -log mu - y / mu
            mu = np.exp(f.eta(L, x)[0])
            np.testing.assert_allclose(f.loglik(L, x), -np.log(mu) - L.y / mu, rtol=1e-13, atol=1e-13)


def test_the_oracle_covers_models_that_mix_old_and_new_factors():
    from oracle import ir_numpy_bounded, ir_numpy_survival

    a, b = ir.survival_regression_ir("weibull", "right_censored", n_obs=50), ir.censored_regression_ir(n_obs=40, n_groups=3)
    L2 = b.likelihoods[0]
    L2.name = "y2"
    off = {v.name for v in a.vars}
    m = ModelIR(vars=a.vars + [v for v in b.vars if v.name not in off],
                priors=a.priors + [p for p in b.priors if p.var not in off], likelihoods=a.likelihoods + [L2])
    f = ir_numpy_survival.make_logp(m)
    q = m.initial_point() + np.random.default_rng(5).uniform(-0.3, 0.3, m.n)
    lp, g = f(q)
    x, _ = f.constrained(q)
    L = m.likelihoods[0]
    want = float(np.sum(f.loglik(L, x))) + ir_numpy_bounded.make_logp(
        ModelIR(vars=m.vars, priors=m.priors, likelihoods=[L2]))(q)[0]
    assert abs(lp - want) <= 1e-12 * abs(want)
    assert np.max(np.abs(fd_grad(f, q) - g)) <= 1e-5 * max(1.0, np.max(np.abs(g)))


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the support rule, lowering, specialise, fuse_design_columns, the sampler's data groups
# ------------------------------------------------------------------------------------------------------------------------
def _one(dist, y, lower=None, upper=None, **slot):
    if not slot:
        slot = {"alpha": 1.5} if dist in ir.WEIBULL_LIKS else {"sigma": 1.0}
    return ModelIR(vars=[Var("b", "b", 1), Var("s_log__", "s", 1, "log")],
                   likelihoods=[Likelihood(dist, np.asarray(y, dtype=np.float64), [Term([("b", None)])], lower=lower,
                                           upper=upper, **slot)])


REFUSALS = [  # (what, dist, y, lower, upper, the words validate() and b200_model_create share)
    ("y_zero", "weibull_log", [1.0, 0.0], None, None, ir.SURV_Y),
    ("y_negative", "lognormal", [1.0, -2.0], None, None, ir.SURV_Y),
    ("y_not_finite", "censored_weibull_log", [1.0, np.inf], None, 5.0, ir.SURV_Y),
    ("lower_negative", "censored_lognormal", [1.0, 2.0], -0.5, None, ir.SURV_SIDES),
    ("lower_plus_inf", "truncated_weibull_log", [1.0, 2.0], np.inf, None, ir.SURV_SIDES),
    ("upper_zero", "censored_weibull_log", [1.0, 2.0], None, np.array([3.0, 0.0]), ir.SURV_SIDES),
    ("nan_bound", "truncated_lognormal", [1.0, 2.0], np.array([0.5, np.nan]), None, ir.SURV_SIDES),
    ("lower_eq_upper", "censored_lognormal", [1.0, 2.0], np.array([1.0, 0.5]), np.array([1.0, 3.0]), ir.BOUND_ORDER),
    ("y_below_lower", "truncated_weibull_log", [1.0, 2.0], 1.5, None, ir.BOUND_Y),
    ("y_above_upper", "censored_weibull_log", [1.0, 2.0], None, np.array([1.5, 1.9]), ir.BOUND_Y),
    ("truncated_open", "truncated_weibull_log", [1.0, 2.0], 0.0, None, ir.SURV_TRUNC_OPEN),
    ("truncated_all_open", "truncated_lognormal", [1.0, 2.0], np.array([0.0, -np.inf]), np.inf, ir.SURV_TRUNC_OPEN),
]


@pytest.mark.parametrize("what,dist,y,lower,upper,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_validate_refuses_each_clause_of_the_support_rule(what, dist, y, lower, upper, msg):
    with pytest.raises(ValueError) as e:
        _one(dist, y, lower, upper).validate()
    assert msg in str(e.value), (what, str(e.value))


def test_validate_refuses_malformed_slots_and_keeps_the_other_refusals():
    for alpha, msg in ((None, "weibull_log needs alpha"), (0.0, "alpha must be a finite constant > 0"),
                       (Ref("b"), "positive support"), (np.ones(2), "alpha must be one constant or a scalar variable")):
        with pytest.raises(ValueError, match=msg):
            _one("weibull_log", [1.0, 2.0], alpha=alpha).validate()
    with pytest.raises(ValueError, match="has no sigma"):
        _one("censored_weibull_log", [1.0, 2.0], upper=2.0, alpha=1.0, sigma=1.0).validate()
    with pytest.raises(ValueError, match="lognormal likelihood needs sigma"):
        _one("lognormal", [1.0, 2.0], sigma=None).validate()
    with pytest.raises(ValueError, match="sigma must be a finite constant > 0"):
        _one("truncated_lognormal", [1.0, 2.0], lower=0.5, sigma=-1.0).validate()
    with pytest.raises(ValueError, match="alpha belongs to the negative_binomial_log / gamma_log likelihoods"):
        _one("lognormal", [1.0, 2.0], sigma=1.0, alpha=2.0).validate()
    with pytest.raises(ValueError, match=ir.SURV_PLAIN):
        _one("weibull_log", [1.0, 2.0], lower=0.5).validate()
    with pytest.raises(ValueError, match="lower / upper belong to the censored_normal / truncated_normal likelihoods"):
        ModelIR(vars=[Var("b", "b", 1)], likelihoods=[Likelihood("normal", np.ones(2), [Term([("b", None)])], sigma=1.0,
                                                                 lower=0.0)]).validate()
    with pytest.raises(ValueError, match="not in the closed set"):  # no Weibull prior
        ModelIR(vars=[Var("b_log__", "b", 1, "log")], priors=[Prior("weibull", "b_log__", (1.0, 1.0))]).validate()
    for dist, lo, hi in (("censored_weibull_log", None, None), ("censored_lognormal", 0.0, np.inf),
                         ("truncated_weibull_log", np.array([0.0, 0.5]), None), ("truncated_lognormal", -np.inf, 5.0)):
        _one(dist, [1.0, 2.0], lo, hi).validate()
    _one("weibull_log", [1.0, 2.0], alpha=Ref("s_log__")).validate()


def test_lowered_tables_hold_the_dist_the_bound_block_and_the_slot():
    for dist, observe, want in (("weibull", "plain", 18), ("lognormal", "plain", 19), ("weibull", "right_censored", 20),
                                ("lognormal", "right_censored", 21), ("exponential", "entry_truncated", 22),
                                ("lognormal", "entry_truncated", 23)):
        m = ir.survival_regression_ir(dist, observe, n_obs=40)
        L = m.likelihoods[0]
        N = len(L.y)
        c_ir, keep = _lib.build_ir(ir.lower(m))
        lik = ctypes.cast(c_ir.liks, ctypes.POINTER(_lib.IrLik))[0]
        assert lik.dist == want == ir.LIK_DISTS[L.dist] and lik.N == N and lik.y_var == 0
        rows = 1 if observe == "plain" else 3
        block = np.ctypeslib.as_array(ctypes.cast(lik.y, ctypes.POINTER(ctypes.c_double)), (rows, N))
        assert np.array_equal(block[0], L.y)
        if rows == 3:
            lo, hi = L.bounds()
            assert np.array_equal(block[1], lo) and np.array_equal(block[2], hi)
        if dist == "exponential":
            assert lik.sigma_kind == ir.SIGMA_CONST and lik.sigma.value == 1.0
        else:
            ref = m.offsets()["sigma_log__" if dist == "lognormal" else "alpha_log__"]
            assert lik.sigma_kind == ir.SIGMA_REF and lik.sigma.kind == 1 and lik.sigma.ref == ref
    low = ir.lower(build("lognormal-plain-const"))
    assert low.liks[0]["sigma_kind"] == ir.SIGMA_CONST and low.liks[0]["sigma_value"] == 0.8
    low = ir.lower(ir.survival_regression_ir("weibull", "plain", alpha=2.5, n_obs=20))
    assert low.liks[0]["sigma_kind"] == ir.SIGMA_CONST and low.liks[0]["sigma_value"] == 2.5


def test_the_example_builder():
    for dist in ("weibull", "exponential", "lognormal"):
        m = ir.survival_regression_ir(dist, "right_censored")
        L = m.likelihoods[0]
        assert 0.25 <= np.mean(L.y == L.upper) <= 0.35 and L.lower is None and np.ndim(L.upper) == 1
        m = ir.survival_regression_ir(dist, "entry_truncated")
        L = m.likelihoods[0]
        assert np.ndim(L.lower) == 1 and np.all(L.y > L.lower) and np.any(L.lower == 0.0) and L.upper is None
        assert ir.survival_regression_ir(dist, "plain").likelihoods[0].dist in ("weibull_log", "lognormal")
    assert ir.survival_regression_ir("exponential").likelihoods[0].alpha == 1.0
    assert isinstance(ir.survival_regression_ir("weibull").likelihoods[0].alpha, Ref)
    assert ir.survival_regression_ir("lognormal", alpha=0.6).likelihoods[0].sigma == 0.6
    with pytest.raises(ValueError):
        ir.survival_regression_ir("exponential", alpha=2.0)


def _as_columns(m):
    """The builders' design term written one column per term, the form from_pymc produces for dot(X, beta)."""
    import copy

    out = copy.deepcopy(m)
    for L in out.likelihoods:
        terms = []
        for t in L.terms:
            if ir.is_design(t):
                X = np.asarray(t.coef)
                terms += [Term([(t.factors[0][0], np.full(len(L.y), k, dtype=np.int32))], coef=X[:, k].copy())
                          for k in range(X.shape[1])]
            else:
                terms.append(t)
        L.terms = terms
    return out


def test_specialise_declines_and_fuse_design_columns_keeps_the_bounds():
    from oracle import ir_numpy_survival

    for dist, observe in (("weibull", "right_censored"), ("lognormal", "entry_truncated"), ("lognormal", "plain")):
        m = ir.survival_regression_ir(dist, observe, n_obs=60)
        assert ir.specialise(m) is None and ir.specialise(m, extended=True) is None
        cols = _as_columns(m)
        fused = ir.fuse_design_columns(cols)
        L, F = m.likelihoods[0], fused.likelihoods[0]
        assert F.dist == L.dist and np.array_equal(F.y, L.y) and sum(ir.is_design(t) for t in F.terms) == 1
        for a, b in ((F.lower, L.lower), (F.upper, L.upper), (F.alpha, L.alpha), (F.sigma, L.sigma)):
            assert (a is None and b is None) or np.array_equal(a, b)
        f, g = ir_numpy_survival.make_logp(fused), ir_numpy_survival.make_logp(cols)
        q = m.initial_point() + np.random.default_rng(3).uniform(-0.5, 0.5, m.n)
        (a, ga), (b, gb) = f(q), g(q)
        assert abs(a - b) <= 1e-12 * abs(b) and np.allclose(ga, gb, rtol=1e-11, atol=1e-11)


def test_sampler_records_the_data_and_the_survival_log_likelihood():
    """The sampler on the oracle-backed stand-in: observed_data keeps y, constant_data the per-observation follow-up
    times, and the log_likelihood group holds log S at the censored observations and log f at the others."""
    from b200_helpers import OracleEngine
    from oracle import ir_numpy_survival
    from pymc_b200 import engine, sampling

    m = ir.survival_regression_ir("weibull", "right_censored", n_obs=60, n_groups=4, seed=5)

    class IrStandIn(OracleEngine):
        def __init__(self, model):
            self.ir, self.spec = model, engine._ir_spec(model)
            self.n, self.f = model.n, ir_numpy_survival.make_logp(model)

        def pointwise_loglik(self, draws, lik=0):
            q = np.asarray(draws)
            L = self.ir.likelihoods[lik]
            out = np.empty(q.shape[:-1] + (len(L.y),))
            for ix in np.ndindex(*q.shape[:-1]):
                out[ix] = self.f.loglik(L, self.f.constrained(q[ix])[0])
            return out

    res = sampling.sample_b200_nuts(5, tune=10, chains=2, random_seed=4, model=IrStandIn(m), momentum="numpy",
                                    keep_untransformed=True, idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
    L = m.likelihoods[0]
    assert np.array_equal(res.constant_data["y_upper"], L.upper) and "y_lower" not in res.constant_data
    assert np.array_equal(res.observed_data["y"], L.y)
    ll = res.log_likelihood["y"]
    assert ll.shape == (2, 5, 60)
    X = L.terms[2].coef
    g = L.terms[1].factors[1][1]
    for c in range(2):
        for d in range(5):
            P = {k: res.posterior[k][c, d] for k in ("b0", "z", "sigma_a", "beta", "alpha")}
            eta = P["b0"] + P["sigma_a"] * P["z"][g] + X @ P["beta"]
            np.testing.assert_allclose(ll[c, d], scipy_pointwise(L, eta, P["alpha"]), rtol=1e-11, atol=1e-11)
            cens = L.y == L.upper
            w = stats.weibull_min(P["alpha"], scale=np.exp(eta[cens]))
            np.testing.assert_allclose(ll[c, d][cens], w.logsf(L.y[cens]), rtol=1e-12, atol=1e-12)


def test_model_create_refuses_malformed_survival_tables_through_the_c_abi():
    """prepare_ir makes the checks of validate(), with the same words, for callers of the C ABI; a survival likelihood is
    not a latent factor."""
    def set_y(row, k, value):
        def edit(low):
            y = low.liks[0]["y"].copy()
            if y.ndim == 1:
                y[k] = value
            else:
                y[row, k] = value
            low.liks[0]["y"] = y
        return edit

    def crossed(low):
        low.liks[0]["y"] = low.liks[0]["y"].copy()
        low.liks[0]["y"][1, 0], low.liks[0]["y"][2, 0] = 2.0, 1.0

    def both_open(low):
        low.liks[0]["y"] = low.liks[0]["y"].copy()
        low.liks[0]["y"][1] = 0.0
        low.liks[0]["y"][2] = np.inf

    w = lambda obs: (lambda: ir.survival_regression_ir("weibull", obs, n_obs=30))  # noqa: E731
    ln = lambda obs: (lambda: ir.survival_regression_ir("lognormal", obs, n_obs=30))  # noqa: E731
    bad_alpha = lambda low: low.liks[0].update(sigma_value=-1.0, sigma_kind=ir.SIGMA_CONST)  # noqa: E731
    obs_alpha = lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_OBS, sigma_obs=np.ones(30))  # noqa: E731
    as_latent = lambda low: low.liks[0].update(y_var=1)  # noqa: E731
    cases = [
        (w("plain"), set_y(0, 0, 0.0), ir.SURV_Y), (ln("plain"), set_y(0, 3, -1.0), ir.SURV_Y),
        (w("right_censored"), set_y(0, 0, np.nan), ir.SURV_Y),
        (w("right_censored"), set_y(1, 0, -0.5), ir.SURV_SIDES), (ln("entry_truncated"), set_y(1, 2, np.inf), ir.SURV_SIDES),
        (ln("right_censored"), set_y(2, 0, 0.0), ir.SURV_SIDES), (w("entry_truncated"), set_y(2, 0, np.nan), ir.SURV_SIDES),
        (w("entry_truncated"), crossed, ir.BOUND_ORDER), (ln("right_censored"), set_y(0, 0, 1e6), ir.BOUND_Y),
        (w("entry_truncated"), both_open, ir.SURV_TRUNC_OPEN), (ln("entry_truncated"), both_open, ir.SURV_TRUNC_OPEN),
        (w("plain"), bad_alpha, "alpha must be a finite constant > 0"), (w("plain"), obs_alpha, "alpha must be a constant or"),
        (ln("plain"), bad_alpha, "sigma must be a finite constant > 0"),
        (w("right_censored"), as_latent, "latent factor"), (ln("entry_truncated"), as_latent, "latent factor"),
    ]
    for builder, edit, msg in cases:
        err = refusal_after_edit(builder, edit)
        assert err is not None and msg in err, (msg, err)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
BUILDERS = {
    "weibull_censored": lambda: ir.survival_regression_ir("weibull", "right_censored"),                 # n = 14: warp
    "weibull_censored_cta": lambda: ir.survival_regression_ir("weibull", "right_censored", n_obs=1500, n_groups=300,
                                                              seed=7),                                  # n = 305: CTA
    "lognormal_truncated": lambda: ir.survival_regression_ir("lognormal", "entry_truncated"),
    "lognormal_truncated_cta": lambda: ir.survival_regression_ir("lognormal", "entry_truncated", n_obs=1200, n_groups=280,
                                                                 seed=8),
    "exponential_truncated": lambda: ir.survival_regression_ir("exponential", "entry_truncated"),
    "weibull_plain_const": lambda: ir.survival_regression_ir("weibull", "plain", alpha=2.0),
    "lognormal_censored": lambda: ir.survival_regression_ir("lognormal", "right_censored"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("cid", CASE_IDS)
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid):
    """Chain = warp, then chain = CTA forced: each against the mp reference and the oracle, bit-identical when repeated."""
    from oracle import ir_numpy_survival
    from pymc_b200 import engine

    m = build(cid)
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = ir_numpy_survival.make_logp(m)
    Q, lp_mp, S, g_mp, G = mp_reference(cid)
    go = np.array([f(q)[1] for q in Q])
    lo = np.array([f(q)[0] for q in Q])
    for team, (lp, g) in logp_at_both_team_shapes(cm, Q).items():
        assert np.all(np.isfinite(lp)) and np.all(np.isfinite(g)), (cid, team)
        assert_close_to_reference(lp, g, lp_mp, S, g_mp, G, (cid, team))
        assert_close_to_reference(lp, g, lo, S, go, G, (cid, team, "oracle"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_device_function_matches_the_oracle_on_the_builders(name):
    from oracle import ir_numpy_survival
    from pymc_b200 import engine

    m = BUILDERS[name]()
    cm = engine.CompiledModel(m)  # default path: no hand kernel takes it
    assert cm.spec.name == "ir" and (m.n > 256) == name.endswith("cta")
    f = ir_numpy_survival.make_logp(m)
    Q = m.initial_point() + np.random.default_rng(0).uniform(-1.0, 1.0, (9, m.n))
    lp, g = cm.logp_dlogp(Q)
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12
    assert np.max(np.abs(g - go) / np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))) <= 1e-12
    lp2, g2 = cm.logp_dlogp(Q)
    assert np.array_equal(lp, lp2) and np.array_equal(g, g2)


@pytest.mark.gpu
@pytest.mark.parametrize("name,eps", [("weibull_censored", 0.05), ("lognormal_truncated", 0.05), ("weibull_censored_cta", 0.01)])
def test_fixed_step_nuts_matches_the_oracle_sampler(name, eps):
    from oracle import ir_numpy_survival

    m = BUILDERS[name]()
    fixed_step_against_oracle(m, ir_numpy_survival.make_logp(m), eps)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle():
    from oracle import ir_numpy_survival

    m = ir.survival_regression_ir("weibull", "entry_truncated")
    fixed_step_against_oracle(m, ir_numpy_survival.make_logp(m), 0.2, dense_cov=random_dense_cov(m.n, 2, 0.02, 0.05, 12),
                              C=2, T=10)


@pytest.mark.gpu
def test_adaptive_censored_weibull_run_matches_the_oracle_posterior():
    """64 device chains against 8 oracle chains (NUTS with diagonal mass adaptation) on the right-censored Weibull with a
    random alpha: posterior means within 5 SE, standard deviations within 25 %, divergences below 2 %."""
    from oracle import ir_numpy_survival

    m = ir.survival_regression_ir("weibull", "right_censored")
    adaptive_against_oracle(m, ir_numpy_survival.make_logp(m), chain_seed=23, spread=1, philox_seed=5, oracle_seed=200,
                            se_bound=5.0, max_divergence=0.02)


def _scipy_on_draws(m, q):
    from oracle import ir_numpy_survival

    f = ir_numpy_survival.make_logp(m)
    L = m.likelihoods[0]
    out = np.empty(q.shape[:-1] + (len(L.y),))
    for ix in np.ndindex(*q.shape[:-1]):
        x, _ = f.constrained(q[ix])
        out[ix] = scipy_pointwise(L, f.eta(L, x)[0], f.param(L, x)[0])
    return out


@pytest.mark.gpu
def test_pointwise_log_likelihood_and_the_log_likelihood_group_match_scipy():
    import pymc_b200
    from pymc_b200 import engine

    for dist, observe in SCIPY_BUILDS:
        m = ir.survival_regression_ir(dist, observe, n_obs=120)
        cm = engine.CompiledModel(m, specialise=False)
        q = m.initial_point() + np.random.default_rng(4).uniform(-0.5, 0.5, (2, 3, m.n))
        ll = cm.pointwise_loglik(q)
        assert ll.shape == (2, 3, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, _scipy_on_draws(m, q), rtol=1e-11, atol=1e-11, err_msg=f"{dist} {observe}")
    for m in (ir.survival_regression_ir("weibull", "right_censored"), ir.survival_regression_ir("lognormal", "entry_truncated")):
        res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, keep_untransformed=True,
                                         idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
        ll = res.log_likelihood["y"]
        assert ll.shape == (4, 20, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, _scipy_on_draws(m, res.unconstrained), rtol=1e-11, atol=1e-11)
        L = m.likelihoods[0]
        side = "y_upper" if L.upper is not None else "y_lower"
        assert np.array_equal(res.constant_data[side], L.upper if L.upper is not None else L.lower)
