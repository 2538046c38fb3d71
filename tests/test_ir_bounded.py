"""Censored and truncated Normal likelihoods of the model IR (``censored_normal``, ``truncated_normal``).

``_mp_logp`` writes the joint log-density with mpmath at 40 digits from the published definitions, with Phi written
through erfc in both tails (``1 - Phi`` would lose every digit in the upper one even at high precision); the gradient is
``mpmath.diff``.  It reads the ``ModelIR`` dataclasses and nothing else of the package or of oracle/.  S = sum |additive
pieces|: logp is compared to 1e-13 S, as in tests/test_ir_closed_set.py; the gradient to 1e-12 max(1, |g|_inf) plus 1e-15 G,
G the reference's sum of the sizes of the parts d logp / d eta is formed from (``_mp_grad_pieces``).

CPU: the reference against scipy.stats, the oracle (oracle/ir_numpy_bounded.py) against the reference on every catalogue
case (standardised bounds from -37 to 37, narrow windows in one tail, mixed open sides, every sigma kind, design terms),
the support rule, the lowered tables, ``specialise`` / ``fuse_design_columns``, and the sampler's data groups through the
oracle-backed stand-in.  GPU: the generic device function against both, the pointwise log-likelihood, fixed-step and
adaptive NUTS against the oracle sampler, and the C ABI's refusals."""
import ctypes
import zlib
from functools import lru_cache

import mpmath
import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import stats
from b200_helpers import (adaptive_against_oracle, fixed_step_against_oracle, logp_at_both_team_shapes, random_dense_cov,
                          refusal_after_edit)
from test_ir_closed_set import GRAD_TOL, LP_TOL, MP_DPS

from pymc_b200 import _lib, ir
from pymc_b200.ir import Likelihood, ModelIR, Prior, Ref, Term, Var


# ------------------------------------------------------------------------------------------------------------------------
# the high-precision reference
# ------------------------------------------------------------------------------------------------------------------------
def _mp_Phi(z):
    return mp.erfc(-z / mp.sqrt(2)) / 2


def _mp_Q(z):
    return mp.erfc(z / mp.sqrt(2)) / 2


def _mp_normal(y, eta, s):
    z = (y - eta) / s
    return [-z * z / 2, -mp.log(s), -mp.log(2 * mp.pi) / 2]


def _mp_lik_pieces(dist, y, eta, s, lo, hi):
    """Pieces of log p(y | eta) of one bounded observation; lo / hi are mpf or +-mp.inf."""
    if dist == "censored_normal":
        if y == lo:
            return [mp.log(_mp_Phi((y - eta) / s))]
        if y == hi:
            return [mp.log(_mp_Q((y - eta) / s))]
        return _mp_normal(y, eta, s)
    a, b = (lo - eta) / s, (hi - eta) / s
    if a >= 0:  # both bounds above the mode: the difference of the upper tails
        Z = _mp_Q(a) - _mp_Q(b)
    else:
        Z = _mp_Phi(b) - _mp_Phi(a)
    return _mp_normal(y, eta, s) + [-mp.log(Z)]


def _mp_constrain(m, q):
    x, jac, o = {}, [], 0
    for v in m.vars:
        qv = q[o : o + v.size]
        o += v.size
        if v.transform == "log":
            x[v.name] = [mp.exp(t) for t in qv]
            jac += [[t] for t in qv]
        elif v.transform == "interval":
            lo, hi = mpf(v.bounds[0]), mpf(v.bounds[1])
            sg = [1 / (1 + mp.exp(-t)) for t in qv]
            x[v.name] = [lo + (hi - lo) * s for s in sg]
            jac += [[mp.log(hi - lo), mp.log(s), mp.log(s) - t] for s, t in zip(sg, qv)]
        else:
            x[v.name] = list(qv)
            jac += [[] for _ in qv]
    return x, jac


def _mp_side(v):
    v = float(v)
    return mp.inf if v == np.inf else (-mp.inf if v == -np.inf else mpf(v))


def _mp_eta(m, L, x):
    """The linear predictor of likelihood L at the constrained values x (variable name -> list of mpf)."""
    name = lambda r: m.var(r).name  # noqa: E731
    N = len(L.y)
    eta = [mpf(0)] * N
    for t in L.terms:
        if ir.is_design(t):
            X = np.asarray(t.coef)
            b = x[name(t.factors[0][0])]
            for i in range(N):
                eta[i] += mp.fsum(mpf(float(X[i, k])) * b[k] for k in range(X.shape[1]))
            continue
        coef = [mpf(1)] * N if t.coef is None else [mpf(float(c)) for c in np.broadcast_to(t.coef, (N,))]
        for i in range(N):
            pr = coef[i]
            for vn, idx in t.factors:
                xv = x[name(vn)]
                pr *= xv[int(idx[i])] if idx is not None else (xv[0] if len(xv) == 1 else xv[i])
            eta[i] += pr
    return eta


def _mp_sigma(m, L, x):
    N = len(L.y)
    if isinstance(L.sigma, Ref):
        return [x[m.var(L.sigma.var).name][0]] * N
    return [mpf(float(v)) for v in np.broadcast_to(L.sigma, (N,))]


def _mp_grad_pieces(m, q):
    """G = sum over observations of |z| / sigma + (phi(a) + phi(b)) / (sigma Z) (phi(zc) / Phi(zc) for a censored one): the
    size of the parts d logp / d eta is summed from, as S is for logp.  A window 1e-3 sd wide far in a tail has ratios of
    ~1 / width that cancel to O(1), so its gradient carries rounding of 1e-16 G, not of 1e-16 |g|."""
    with mp.workdps(MP_DPS):
        x, _ = _mp_constrain(m, [mpf(float(t)) for t in q])
        G = mpf(0)
        for L in m.likelihoods:
            eta, sg = _mp_eta(m, L, x), _mp_sigma(m, L, x)
            lo_, hi_ = L.bounds()
            for i in range(len(L.y)):
                y, s, lo, hi = mpf(float(L.y[i])), sg[i], _mp_side(lo_[i]), _mp_side(hi_[i])
                z = (y - eta[i]) / s
                G += abs(z) / s
                if L.dist == "censored_normal":
                    if y == lo or y == hi:
                        zc = z if y == lo else -z
                        G += mp.npdf(zc) / _mp_Phi(zc) / s
                    continue
                a, b = (lo - eta[i]) / s, (hi - eta[i]) / s
                Z = _mp_Q(a) - _mp_Q(b) if a >= 0 else _mp_Phi(b) - _mp_Phi(a)
                G += ((0 if a == -mp.inf else mp.npdf(a)) + (0 if b == mp.inf else mp.npdf(b))) / (s * Z)
        return float(G)


def _mp_factors(m):
    name = lambda r: m.var(r).name  # noqa: E731
    par = lambda a, x: x[name(a.var)][0] if isinstance(a, Ref) else mpf(float(a))  # noqa: E731
    out = []
    for p in m.priors:
        vn = name(p.var)

        def prior(x, p=p, vn=vn):
            a = [par(t, x) for t in p.params]
            if p.dist == "normal":
                return [t for xi in x[vn] for t in _mp_normal(xi, a[0], a[1])]
            if p.dist == "halfnormal":
                return [t for xi in x[vn] for t in _mp_normal(xi, mpf(0), a[0]) + [mp.log(2)]]
            assert p.dist == "uniform"
            return [-mp.log(a[1] - a[0]) for _ in x[vn]]
        out.append(({vn} | {name(a.var) for a in p.params if isinstance(a, Ref)}, prior))
    for L in m.likelihoods:
        N = len(L.y)
        y = [mpf(float(v)) for v in L.y]
        lo_, hi_ = L.bounds()
        lo, hi = [_mp_side(v) for v in lo_], [_mp_side(v) for v in hi_]
        deps = set()
        eta_of = (lambda x, L=L: _mp_eta(m, L, x))
        for t in L.terms:
            deps |= {name(vn) for vn, _ in t.factors}
        sobs = None if isinstance(L.sigma, Ref) or np.ndim(L.sigma) == 0 else [mpf(float(v)) for v in L.sigma]

        def lik(x, L=L, y=y, lo=lo, hi=hi, N=N, sobs=sobs, eta_of=eta_of):
            eta = eta_of(x)
            s = sobs if sobs is not None else [par(L.sigma, x)] * N
            return [t for i in range(N) for t in _mp_lik_pieces(L.dist, y[i], eta[i], s[i], lo[i], hi[i])]
        if isinstance(L.sigma, Ref):
            deps.add(name(L.sigma.var))
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


# ------------------------------------------------------------------------------------------------------------------------
# the case catalogue
# ------------------------------------------------------------------------------------------------------------------------
SIGMAS = {"const": lambda N, rng: 0.9, "ref_log": lambda N, rng: Ref("s_log__"), "ref_int": lambda N, rng: Ref("w_interval__"),
          "obs": lambda N, rng: rng.uniform(0.5, 1.5, N)}


def _sigma_vars(kind):
    if kind == "ref_log":
        return [Var("s_log__", "s", 1, "log")], [Prior("halfnormal", "s_log__", (1.5,))]
    if kind == "ref_int":
        return [Var("w_interval__", "w", 1, "interval", (0.2, 3.0))], [Prior("uniform", "w_interval__", (0.2, 3.0))]
    return [], []


def _regression_case(dist, sigma, shape, rng, N=14):
    """b0 + b1 x (+ a group effect, or as a design term) under a bounded likelihood with bounds of the given shape."""
    x = rng.standard_normal(N)
    eta = 0.3 + 0.8 * x
    y = eta + rng.standard_normal(N)
    vars_ = [Var("b0", "b0", 1), Var("b1", "b1", 1)]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "b1", (0.0, 1.0))]
    terms = [Term([("b0", None)]), Term([("b1", None)], coef=x)]
    if shape == "design":
        X = np.column_stack([np.ones(N), x, rng.standard_normal(N)])
        vars_ = [Var("beta", "beta", 3), Var("g", "g", 3)]
        priors = [Prior("normal", "beta", (0.0, 1.5)), Prior("normal", "g", (0.0, 1.0))]
        terms = [Term([("beta", None)], coef=X), Term([("g", np.arange(N, dtype=np.int32) % 3)])]
    sv, sp = _sigma_vars(sigma)
    vars_, priors = vars_ + sv, priors + sp
    q = np.sort(y)
    if shape in ("const", "design"):
        lower, upper = float(q[2]), float(q[-3])
    elif shape == "lower":
        lower, upper = float(q[3]), None
    elif shape == "upper_array":
        lower, upper = None, np.where(rng.random(N) < 0.5, y + rng.uniform(0.0, 1.0, N), np.inf)
    else:  # "mixed": per-observation bounds with open sides mixed in one array
        lower = np.where(rng.random(N) < 0.5, y - rng.uniform(0.0, 1.5, N), -np.inf)
        upper = np.where(rng.random(N) < 0.5, y + rng.uniform(0.0, 1.5, N), np.inf)
    if dist == "censored_normal":
        lo = np.broadcast_to(-np.inf if lower is None else lower, (N,)).copy()
        hi = np.broadcast_to(np.inf if upper is None else upper, (N,)).copy()
        y = np.clip(y, lo, hi)
        if shape in ("mixed", "upper_array"):  # some observations exactly at a bound of their own
            k = rng.choice(N, 4, replace=False)
            hi[k[2:]] = y[k[2:]]
            lo[k[2:]] = np.minimum(lo[k[2:]], y[k[2:]] - 1.0)
            if shape == "mixed":
                lo[k[:2]] = y[k[:2]]
                hi[k[:2]] = np.maximum(hi[k[:2]], y[k[:2]] + 1.0)
                lower = lo
            upper = hi
    else:  # truncated: y strictly inside
        lo = -np.inf if lower is None else np.broadcast_to(lower, (N,))
        hi = np.inf if upper is None else np.broadcast_to(upper, (N,))
        y = np.clip(y, np.nextafter(lo, np.inf), np.nextafter(hi, -np.inf))
    L = Likelihood(dist, y, terms, sigma=SIGMAS[sigma](N, rng), lower=lower, upper=upper)
    return ModelIR(vars=vars_, priors=priors, likelihoods=[L])


def _tail_case(dist):
    """eta = b0, sigma = 1: at b0 = 0 the standardised bounds sit from -37 to 37, and the truncated windows are 1e-3 to
    1 sd wide with both bounds in one tail."""
    if dist == "censored_normal":
        y = np.array([-37.0, -30.0, -20.0, -8.0, -1.5, -0.2, 0.3, 1.2, 8.0, 20.0, 30.0, 37.0, 0.0, 2.0])
        lower = np.array([-37.0, -30.0, -20.0, -8.0, -1.5, -0.2, -np.inf, -np.inf, -np.inf, -np.inf, -np.inf, -np.inf, -5.0, -np.inf])
        upper = np.array([np.inf] * 6 + [0.3, 1.2, 8.0, 20.0, 30.0, 37.0, np.inf, 5.0])
    else:
        lower = np.array([-37.0, -30.0, -20.0, -3.0, 0.5, 2.0, 19.0, 29.999, 36.999, -0.0005, -np.inf, 25.0])
        upper = np.array([-36.999, -29.0, -19.99, -2.0, 0.501, 3.0, 20.0, 30.0, 37.0, 0.0005, -36.0, np.inf])
        y = np.where(np.isfinite(lower), lower, upper) + 0.5 * np.where(np.isfinite(upper) & np.isfinite(lower), upper - lower, 0.0)
        y[10], y[11] = -36.5, 26.0
    return ModelIR(vars=[Var("b0", "b0", 1)], priors=[Prior("normal", "b0", (0.0, 3.0))],
                   likelihoods=[Likelihood(dist, y, [Term([("b0", None)])], sigma=1.0, lower=lower, upper=upper)])


CASES = {}
for _d, _short in (("censored_normal", "cens"), ("truncated_normal", "trunc")):
    for _s, _sh in (("const", "const"), ("ref_log", "lower"), ("ref_int", "mixed"), ("obs", "upper_array"), ("ref_log", "design"),
                    ("obs", "mixed")):
        CASES[f"{_short}-{_sh}-{_s}"] = (lambda rng, d=_d, s=_s, sh=_sh: _regression_case(d, s, sh, rng))
    CASES[f"{_short}-tails"] = (lambda rng, d=_d: _tail_case(d))
CASE_IDS = list(CASES)


def build(cid):
    return CASES[cid](np.random.default_rng(zlib.crc32(cid.encode())))


def points(m, cid):
    """The initial point + U(-1, 1) (twice); for the tail cases b0 in {-7, 0, 7} as well, which takes the standardised
    bounds past +-37 on one side."""
    rng = np.random.default_rng(zlib.crc32(cid.encode()) + 1)
    q0 = m.initial_point()
    Q = [q0 + rng.uniform(-1.0, 1.0, m.n) for _ in range(2)]
    if cid.endswith("tails"):
        Q += [np.array([b]) for b in (0.0, -0.7, 0.7)]
    return np.array(Q)


@lru_cache(maxsize=None)
def mp_reference(cid):
    m = build(cid)
    Q = points(m, cid)
    lp, S = np.array([_mp_logp(m, q) for q in Q]).T
    return Q, lp, S, np.array([_mp_grad(m, q) for q in Q]), np.array([_mp_grad_pieces(m, q) for q in Q])


def assert_close_to_reference(lp, g, ref_lp, S, ref_g, G, what):
    """logp to 1e-13 S; the gradient to 1e-12 max(1, |g|_inf) plus 1e-15 G (a few ulps of each part it is summed from)."""
    assert np.all(np.abs(lp - ref_lp) <= LP_TOL * S), (what, np.abs(lp - ref_lp) / S)
    err = np.max(np.abs(g - ref_g), axis=1)
    assert np.all(err <= GRAD_TOL * np.maximum(1.0, np.max(np.abs(ref_g), axis=1)) + 1e-15 * G), (what, err, G)


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference and the oracle
# ------------------------------------------------------------------------------------------------------------------------
def test_mp_pieces_equal_scipy():
    rows_c = [(-37.0, 0.0, 1.0), (-3.0, 0.5, 2.0), (0.4, -0.2, 0.7), (6.0, 0.0, 1.0), (37.0, 0.0, 1.0), (12.0, -1.0, 0.4)]
    with mp.workdps(MP_DPS):
        for y, eta, s in rows_c:
            z = (y - eta) / s
            for lo, hi, want in ((y, mp.inf, stats.norm.logcdf(z)), (-mp.inf, y, stats.norm.logsf(z)),
                                 (-mp.inf, mp.inf, stats.norm.logpdf(y, eta, s))):
                got = float(mp.fsum(_mp_lik_pieces("censored_normal", mpf(y), mpf(eta), mpf(s), _mp_side(lo), _mp_side(hi))))
                assert abs(got - want) <= 1e-13 * max(1.0, abs(want)), (y, eta, s, got, want)
        for y, eta, s, lo, hi in [(0.3, 0.0, 1.0, -1.0, 2.0), (1.5, 0.2, 0.8, 1.0, np.inf), (-2.0, 1.0, 1.5, -np.inf, -1.0),
                                  (4.2, 0.0, 1.0, 4.0, 4.5), (-4.2, 0.0, 1.0, -4.5, -4.0), (10.3, 0.0, 1.0, 10.0, 11.0)]:
            want = stats.truncnorm.logpdf(y, (lo - eta) / s, (hi - eta) / s, loc=eta, scale=s)
            got = float(mp.fsum(_mp_lik_pieces("truncated_normal", mpf(y), mpf(eta), mpf(s), _mp_side(lo), _mp_side(hi))))
            assert abs(got - want) <= 1e-12 * max(1.0, abs(want)), (y, lo, hi, got, want)


def test_the_catalogue_covers_the_bounded_forms():
    seen = set()
    for cid in CASE_IDS:
        m = build(cid)
        m.validate()
        L = m.likelihoods[0]
        lo, hi = L.bounds()
        kind = "ref" if isinstance(L.sigma, Ref) else ("obs" if np.ndim(L.sigma) == 1 else "const")
        seen.add((L.dist, kind))
        seen.add((L.dist, "open_mixed")) if (np.any(np.isinf(lo)) and np.any(np.isfinite(lo))) else None
        seen.add((L.dist, "design")) if any(ir.is_design(t) for t in L.terms) else None
        if L.dist == "censored_normal":
            assert np.any((L.y == lo) | (L.y == hi)) and np.any((L.y > lo) & (L.y < hi)), cid
            seen.add((L.dist, "both_sides")) if np.any(L.y == lo) and np.any(L.y == hi) else None
    assert {(d, k) for d in ir.BOUNDED_LIKS for k in ("const", "ref", "obs", "open_mixed", "design")} <= seen
    assert ("censored_normal", "both_sides") in seen
    m = build("trunc-tails")  # both bounds in one tail, down to 1e-3 sd, out to |z| = 37
    lo, hi = m.likelihoods[0].bounds()
    two = np.isfinite(lo) & np.isfinite(hi)
    assert np.min((hi - lo)[two]) <= 1e-3 and np.max(np.abs(lo[np.isfinite(lo)])) >= 37 and np.any(two & (lo > 20))


@pytest.mark.parametrize("cid", CASE_IDS)
def test_oracle_matches_the_mp_reference(cid):
    from oracle import ir_numpy_bounded

    m = build(cid)
    f = ir_numpy_bounded.make_logp(m)
    Q, lp_mp, S, g_mp, G = mp_reference(cid)
    lp, g = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    assert_close_to_reference(lp, g, lp_mp, S, g_mp, G, cid)


def test_oracle_pointwise_equals_scipy_on_the_builders():
    from oracle import ir_numpy_bounded

    for m in (ir.censored_regression_ir(), ir.truncated_regression_ir()):
        f = ir_numpy_bounded.make_logp(m)
        q = m.initial_point() + np.random.default_rng(2).uniform(-0.5, 0.5, m.n)
        x, _ = f.constrained(q)
        L = m.likelihoods[0]
        eta, _ = f.eta(L, x)
        sg, _ = f.sigma(L, x)
        np.testing.assert_allclose(ir_numpy_bounded.bounded_loglik(L, eta, sg), scipy_pointwise(L, eta, sg), rtol=1e-12, atol=1e-12)


def scipy_pointwise(L, eta, sg):
    """log p(y_i | eta_i) of a bounded likelihood from scipy.stats."""
    y = np.asarray(L.y, dtype=np.float64)
    lo, hi = L.bounds()
    if L.dist == "censored_normal":
        return np.where(y == lo, stats.norm.logcdf(y, eta, sg), np.where(y == hi, stats.norm.logsf(y, eta, sg),
                                                                        stats.norm.logpdf(y, eta, sg)))
    return stats.truncnorm.logpdf(y, (lo - eta) / sg, (hi - eta) / sg, loc=eta, scale=sg)


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the support rule, lowering, specialise, fuse_design_columns, the sampler's data groups
# ------------------------------------------------------------------------------------------------------------------------
def _one(dist, y, lower=None, upper=None, sigma=1.0, vars_=None):
    return ModelIR(vars=vars_ or [Var("b", "b", 1)],
                   likelihoods=[Likelihood(dist, np.asarray(y, dtype=np.float64), [Term([("b", None)])], sigma=sigma,
                                           lower=lower, upper=upper)])


REFUSALS = [  # (what, dist, y, lower, upper, the words validate() and b200_model_create share)
    ("lower_plus_inf", "censored_normal", [1.0, 2.0], np.inf, None, ir.BOUND_SIDES),
    ("upper_minus_inf", "truncated_normal", [1.0, 2.0], None, -np.inf, ir.BOUND_SIDES),
    ("nan_bound", "censored_normal", [1.0, 2.0], np.array([0.0, np.nan]), None, ir.BOUND_SIDES),
    ("lower_eq_upper", "censored_normal", [1.0, 2.0], np.array([1.0, 0.0]), np.array([1.0, 3.0]), ir.BOUND_ORDER),
    ("lower_gt_upper", "truncated_normal", [1.0, 2.0], 3.0, 0.0, ir.BOUND_ORDER),
    ("y_below_lower", "censored_normal", [1.0, 2.0], 1.5, None, ir.BOUND_Y),
    ("y_above_upper", "truncated_normal", [1.0, 2.0], None, np.array([1.5, 1.9]), ir.BOUND_Y),
    ("y_not_finite", "censored_normal", [1.0, np.inf], 0.0, None, ir.BOUND_Y),
    ("truncated_unbounded", "truncated_normal", [1.0, 2.0], None, None, ir.TRUNC_OPEN),
    ("truncated_all_open", "truncated_normal", [1.0, 2.0], np.array([-np.inf, -np.inf]), np.inf, ir.TRUNC_OPEN),
]


@pytest.mark.parametrize("what,dist,y,lower,upper,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_validate_refuses_each_clause_of_the_support_rule(what, dist, y, lower, upper, msg):
    with pytest.raises(ValueError) as e:
        _one(dist, y, lower, upper).validate()
    assert msg in str(e.value), (what, str(e.value))


def test_validate_refuses_malformed_bound_slots_and_misplaced_bounds():
    for lower in (np.zeros(3), np.zeros((2, 1)), Ref("b")):
        with pytest.raises(ValueError, match="lower and upper"):
            _one("censored_normal", [1.0, 2.0], lower=lower).validate()
    with pytest.raises(ValueError, match="belong to the censored_normal"):
        _one("normal", [1.0, 2.0], lower=0.0).validate()
    with pytest.raises(ValueError, match="needs sigma"):
        _one("truncated_normal", [1.0, 2.0], lower=0.0, sigma=None).validate()
    with pytest.raises(ValueError, match="sigma must be a finite constant > 0"):
        _one("censored_normal", [1.0, 2.0], lower=0.0, sigma=-1.0).validate()
    with pytest.raises(ValueError, match="positive support"):
        _one("truncated_normal", [1.0, 2.0], lower=0.0, sigma=Ref("b")).validate()
    with pytest.raises(ValueError, match="not in the closed set"):  # no bounded prior: these are likelihoods only
        ModelIR(vars=[Var("b", "b", 1)], priors=[Prior("censored_normal", "b", (0.0, 1.0))]).validate()
    for dist, lower, upper in (("censored_normal", None, None), ("censored_normal", -np.inf, np.inf), ("truncated_normal", 0.0, None),
                               ("truncated_normal", np.array([-np.inf, 0.0]), np.array([np.inf, np.inf]))):
        _one(dist, [1.0, 2.0], lower, upper).validate()


def test_lowered_tables_hold_the_dist_the_bound_block_and_the_sigma_slot():
    for m, dist_id in ((ir.censored_regression_ir(), 8), (ir.truncated_regression_ir(), 9)):
        c_ir, keep = _lib.build_ir(ir.lower(m))
        lik = ctypes.cast(c_ir.liks, ctypes.POINTER(_lib.IrLik))[0]
        L = m.likelihoods[0]
        N = len(L.y)
        block = np.ctypeslib.as_array(ctypes.cast(lik.y, ctypes.POINTER(ctypes.c_double)), (3, N))
        lo, hi = L.bounds()
        assert lik.dist == dist_id == ir.LIK_DISTS[L.dist] and lik.N == N and lik.y_var == 0
        assert np.array_equal(block[0], L.y) and np.array_equal(block[1], lo) and np.array_equal(block[2], hi)
        assert lik.sigma_kind == ir.SIGMA_REF and lik.sigma.kind == 1 and lik.sigma.ref == m.offsets()["sigma_log__"]
    m = build("cens-upper_array-obs")
    low = ir.lower(m)
    assert low.liks[0]["sigma_kind"] == ir.SIGMA_OBS and np.array_equal(low.liks[0]["sigma_obs"], m.likelihoods[0].sigma)
    assert np.all(np.isneginf(low.liks[0]["y"][1])) and ir.lower(build("cens-const-const")).liks[0]["sigma_kind"] == ir.SIGMA_CONST


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
    from oracle import ir_numpy_bounded

    for m in (ir.censored_regression_ir(), ir.truncated_regression_ir()):
        assert ir.specialise(m) is None and ir.specialise(m, extended=True) is None
        cols = _as_columns(m)
        fused = ir.fuse_design_columns(cols)
        L, F = m.likelihoods[0], fused.likelihoods[0]
        assert F.dist == L.dist and F.lower == L.lower and np.array_equal(F.upper, L.upper) and np.array_equal(F.y, L.y)
        assert sum(ir.is_design(t) for t in F.terms) == 1
        f, g = ir_numpy_bounded.make_logp(fused), ir_numpy_bounded.make_logp(cols)
        q = m.initial_point() + np.random.default_rng(3).uniform(-0.5, 0.5, m.n)
        (a, ga), (b, gb) = f(q), g(q)
        assert abs(a - b) <= 1e-12 * abs(b) and np.allclose(ga, gb, rtol=1e-11, atol=1e-11)


def test_sampler_records_the_bounds_and_the_censored_log_likelihood():
    """Seam B4 on the oracle-backed stand-in: constant_data holds the per-observation bounds; the log_likelihood group
    holds log Phi / log(1 - Phi) for the censored observations and the Normal log-density for the others."""
    from b200_helpers import OracleEngine
    from oracle import ir_numpy_bounded
    from pymc_b200 import engine, sampling

    m = ir.censored_regression_ir(n_obs=60, n_groups=4, seed=5)

    class IrStandIn(OracleEngine):
        def __init__(self, model):
            self.ir, self.spec = model, engine._ir_spec(model)
            self.n, self.f = model.n, ir_numpy_bounded.make_logp(model)

        def pointwise_loglik(self, draws, lik=0):
            q = np.asarray(draws)
            out = np.empty(q.shape[:-1] + (len(self.ir.likelihoods[lik].y),))
            for ix in np.ndindex(*q.shape[:-1]):
                x, _ = self.f.constrained(q[ix])
                L = self.ir.likelihoods[lik]
                out[ix] = ir_numpy_bounded.bounded_loglik(L, self.f.eta(L, x)[0], self.f.sigma(L, x)[0])
            return out

    res = sampling.sample_b200_nuts(5, tune=10, chains=2, random_seed=4, model=IrStandIn(m), momentum="numpy",
                                    keep_untransformed=True, idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
    L = m.likelihoods[0]
    assert np.array_equal(res.constant_data["y_upper"], L.upper) and "y_lower" not in res.constant_data  # lower: one constant
    assert np.array_equal(res.observed_data["y"], L.y)
    ll = res.log_likelihood["y"]
    assert ll.shape == (2, 5, 60)
    lo, hi = L.bounds()
    X = L.terms[1].coef
    g = L.terms[0].factors[0][1]
    for c in range(2):
        for d in range(5):
            eta = res.posterior["a"][c, d][g] + X @ res.posterior["beta"][c, d]
            sg = res.posterior["sigma"][c, d]
            want = scipy_pointwise(L, eta, sg)
            np.testing.assert_allclose(ll[c, d], want, rtol=1e-12, atol=1e-12)
            assert np.all(ll[c, d][L.y == lo] == stats.norm.logcdf(lo[L.y == lo], eta[L.y == lo], sg))  # left-censored


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
BUILDERS = {
    "censored": ir.censored_regression_ir,                                              # n = 14: chain = warp
    "censored_cta": lambda: ir.censored_regression_ir(n_obs=1500, n_groups=300, seed=7),  # n = 306: chain = CTA
    "truncated": ir.truncated_regression_ir,
    "truncated_cta": lambda: ir.truncated_regression_ir(n_obs=1200, n_features=260, seed=8),  # n = 262
}


@pytest.mark.gpu
@pytest.mark.parametrize("cid", CASE_IDS)
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid):
    """Chain = warp, then chain = CTA forced: each against the mp reference and the oracle, bit-identical when repeated."""
    from oracle import ir_numpy_bounded
    from pymc_b200 import engine

    m = build(cid)
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = ir_numpy_bounded.make_logp(m)
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
    from oracle import ir_numpy_bounded
    from pymc_b200 import engine

    m = BUILDERS[name]()
    cm = engine.CompiledModel(m)  # default path: no hand kernel takes it; the design term runs as written
    assert cm.spec.name == "ir" and (m.n > 256) == name.endswith("cta")
    f = ir_numpy_bounded.make_logp(m)
    Q = m.initial_point() + np.random.default_rng(0).uniform(-1.0, 1.0, (9, m.n))
    lp, g = cm.logp_dlogp(Q)
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12
    assert np.max(np.abs(g - go) / np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))) <= 1e-12
    lp2, g2 = cm.logp_dlogp(Q)
    assert np.array_equal(lp, lp2) and np.array_equal(g, g2)


@pytest.mark.gpu
@pytest.mark.parametrize("name,eps", [("censored", 0.05), ("truncated", 0.05), ("censored_cta", 0.01)])
def test_fixed_step_nuts_matches_the_oracle_sampler(name, eps):
    from oracle import ir_numpy_bounded

    m = BUILDERS[name]()
    fixed_step_against_oracle(m, ir_numpy_bounded.make_logp(m), eps)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle():
    from oracle import ir_numpy_bounded

    m = ir.truncated_regression_ir()
    fixed_step_against_oracle(m, ir_numpy_bounded.make_logp(m), 0.3, dense_cov=random_dense_cov(m.n, 2, 0.02, 0.05, 12),
                              C=2, T=10)


@pytest.mark.gpu
def test_adaptive_censored_run_matches_the_oracle_posterior():
    """64 device chains against 8 oracle chains (NUTS with diagonal mass adaptation) on the censored regression: posterior
    means within 5 SE, standard deviations within 25 %, divergences below 2 %."""
    from oracle import ir_numpy_bounded

    m = ir.censored_regression_ir()
    adaptive_against_oracle(m, ir_numpy_bounded.make_logp(m), specialise=True, chain_seed=23, spread=1, philox_seed=5,
                            oracle_seed=200, se_bound=5.0, max_divergence=0.02)


def _scipy_on_draws(m, q):
    from oracle import ir_numpy_bounded

    f = ir_numpy_bounded.make_logp(m)
    L = m.likelihoods[0]
    out = np.empty(q.shape[:-1] + (len(L.y),))
    for ix in np.ndindex(*q.shape[:-1]):
        x, _ = f.constrained(q[ix])
        out[ix] = scipy_pointwise(L, f.eta(L, x)[0], f.sigma(L, x)[0])
    return out


@pytest.mark.gpu
def test_pointwise_log_likelihood_and_the_log_likelihood_group_match_scipy():
    import pymc_b200
    from pymc_b200 import engine

    for cid in ("cens-mixed-obs", "trunc-mixed-ref_int", "cens-tails", "trunc-upper_array-obs"):
        m = build(cid)
        cm = engine.CompiledModel(m, specialise=False)
        q = m.initial_point() + np.random.default_rng(4).uniform(-0.5, 0.5, (2, 3, m.n))
        ll = cm.pointwise_loglik(q)
        assert ll.shape == (2, 3, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, _scipy_on_draws(m, q), rtol=1e-12, atol=1e-12, err_msg=cid)
    for m in (ir.censored_regression_ir(), ir.truncated_regression_ir()):
        res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, keep_untransformed=True,
                                         idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
        ll = res.log_likelihood["y"]
        assert ll.shape == (4, 20, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, _scipy_on_draws(m, res.unconstrained), rtol=1e-12, atol=1e-12)
        assert np.array_equal(res.constant_data["y_upper"], m.likelihoods[0].upper)


def test_model_create_refuses_malformed_bound_tables_through_the_c_abi():
    """prepare_ir makes the checks of validate(), with the same words, for callers of the C ABI; a bounded Normal is not a
    latent factor."""
    def set_y(row, k, value):
        def edit(low):
            low.liks[0]["y"] = low.liks[0]["y"].copy()
            low.liks[0]["y"][row, k] = value
        return edit

    def both_open(low):
        low.liks[0]["y"] = low.liks[0]["y"].copy()
        low.liks[0]["y"][1] = -np.inf
        low.liks[0]["y"][2] = np.inf

    c, t = ir.censored_regression_ir, ir.truncated_regression_ir
    bad_sigma = lambda low: low.liks[0].update(sigma_value=-1.0, sigma_kind=ir.SIGMA_CONST)  # noqa: E731
    as_latent = lambda low: low.liks[0].update(y_var=1)  # noqa: E731  (a latent factor on its first variable)
    cases = [
        (c, set_y(1, 0, np.inf), ir.BOUND_SIDES), (t, set_y(2, 0, -np.inf), ir.BOUND_SIDES),
        (c, set_y(2, 3, np.nan), ir.BOUND_SIDES), (c, set_y(2, 0, -100.0), ir.BOUND_ORDER), (t, set_y(2, 0, -1.0), ir.BOUND_ORDER),
        (c, set_y(0, 0, -100.0), ir.BOUND_Y), (t, set_y(0, 0, -1.0), ir.BOUND_Y), (c, set_y(0, 1, np.nan), ir.BOUND_Y),
        (t, both_open, ir.TRUNC_OPEN),
        (c, bad_sigma, "must be a finite constant > 0"), (t, bad_sigma, "must be a finite constant > 0"),
        (c, as_latent, "latent factor"), (t, as_latent, "latent factor"),
    ]
    for builder, edit, msg in cases:
        err = refusal_after_edit(builder, edit)
        assert err is not None and msg in err, (msg, err)
