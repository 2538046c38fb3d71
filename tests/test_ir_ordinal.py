"""Ordinal likelihoods (``ordered_logistic``, ``ordered_probit``) and the ordered transform of the model IR.

``_mp_lik`` writes log p(y | eta) of one ordinal observation with mpmath at 40 digits from the published definitions
(OrderedLogistic / OrderedProbit.compute_p, pymc/distributions/discrete.py:1312-1326, :1416-1432, read by
Categorical.logp, :1190-1206), taking the difference of the two CDFs on the side of the mode where it does not cancel.
``_mp_logp`` is the joint log-density of a catalogue model (the ordered transform restated from transforms.py:96-120).
S = sum |additive pieces|; logp is compared to 1e-13 S as in tests/test_ir_closed_set.py.  The probit link forms its window
from two standardised bounds, so it also carries 1e-15 sum (|a| + |b| + 1) / (b - a) of rounding (``_conditioning``).

CPU: the reference against scipy and the reference's own known answers, the oracle (oracle/ir_numpy_ordinal.py) against it
on the catalogue and against central differences, the K = 2 identities, the ordered transform, the support rule and the
lowered tables.  GPU: the generic device function against both, fixed-step and adaptive NUTS against the oracle sampler,
the pointwise log-likelihood and the C ABI's refusals."""
import zlib
from functools import lru_cache

import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import special, stats
from b200_helpers import (adaptive_against_oracle, fd_grad, fixed_step_against_oracle, logp_at_both_team_shapes, random_dense_cov,
                          refusal_after_edit)
from test_ir_closed_set import LP_TOL, MP_DPS

from pymc_b200 import ir, models
from pymc_b200.ir import Likelihood, ModelIR, Prior, Ref, Term, Var


def oracle(m):
    from ir_latent_oracle import make_logp as latent
    from oracle import ir_numpy_ordinal

    return ir_numpy_ordinal.make_logp(m, base=latent)


# ------------------------------------------------------------------------------------------------------------------------
# the high-precision reference
# ------------------------------------------------------------------------------------------------------------------------
def _mp_F(link, t):
    if link == "ordered_logistic":
        return 1 / (1 + mp.exp(-t))
    return mp.erfc(-t / mp.sqrt(2)) / 2


def _mp_lik(link, y, K, eta, s, c):
    """log p(y | eta) of one observation; c: the K - 1 cutpoints (mpf)."""
    a = (c[y - 1] - eta) / s if y > 0 else -mp.inf
    b = (c[y] - eta) / s if y < K - 1 else mp.inf
    F = lambda t: mpf(0) if t == -mp.inf else (mpf(1) if t == mp.inf else _mp_F(link, t))  # noqa: E731
    G = lambda t: F(-t) if abs(t) != mp.inf else 1 - F(t)  # 1 - F(t), the upper tail  # noqa: E731
    return mp.log(G(a) - G(b)) if a > 0 else mp.log(F(b) - F(a))


def _mp_constrain(m, q):
    x, jac, o = {}, [], 0
    for v in m.vars:
        qv = [mpf(float(t)) for t in q[o : o + v.size]]
        o += v.size
        if v.transform == "log":
            x[v.name] = [mp.exp(t) for t in qv]
            jac += qv
        elif v.transform in ir.ORDERED_TRANSFORMS:  # Ordered.backward / log_jac_det, transforms.py:96-120
            pos = v.transform == "ordered_positive"
            d = [mp.exp(t) for t in qv] if pos else [qv[0]] + [mp.exp(t) for t in qv[1:]]
            x[v.name] = [mp.fsum(d[: k + 1]) for k in range(len(d))]
            jac += qv if pos else qv[1:]
        else:
            x[v.name] = qv
    return x, jac


def _mp_eta(m, L, x):
    from test_ir_bounded import _mp_eta as eta

    return eta(m, L, x)


def _mp_scale(m, L, x, N):
    if L.dist == "ordered_logistic":
        return [mpf(1)] * N
    if isinstance(L.sigma, Ref):
        return [x[m.var(L.sigma.var).name][0]] * N
    return [mpf(float(v)) for v in np.broadcast_to(L.sigma, (N,))]


def _mp_cut(m, L, x):
    return x[m.var(L.cutpoints.var).name] if isinstance(L.cutpoints, Ref) else [mpf(float(c)) for c in L.cutpoints]


def _mp_logp(m, q):
    """(logp, S) of a catalogue model: normal / halfnormal priors with constant parameters, ordinal likelihoods."""
    with mp.workdps(MP_DPS):
        x, pieces = _mp_constrain(m, q)
        for p in m.priors:
            xs = x[m.var(p.var).name]
            if p.dist == "normal":
                mu, sd = (mpf(float(t)) for t in p.params)
                pieces += [t for xi in xs for t in (-((xi - mu) / sd) ** 2 / 2, -mp.log(sd), -mp.log(2 * mp.pi) / 2)]
            else:
                assert p.dist == "halfnormal"
                sd = mpf(float(p.params[0]))
                pieces += [t for xi in xs for t in (-(xi / sd) ** 2 / 2, -mp.log(sd), mp.log(2 / mp.pi) / 2)]
        for L in m.likelihoods:
            N = len(L.y)
            K = L.n_categories(m)
            eta, s, c = _mp_eta(m, L, x), _mp_scale(m, L, x, N), _mp_cut(m, L, x)
            pieces += [_mp_lik(L.dist, int(L.y[i]), K, eta[i], s[i], c) for i in range(N)]
        return float(mp.fsum(pieces)), float(mp.fsum(abs(t) for t in pieces))


def _conditioning(m, q, power=1):
    """sum over probit observations of (|a| + |b| + 1) / (b - a)^power: the rounding of forming the window from two bounds,
    in log Z (power 1) and in phi / Z, which the gradient carries (power 2)."""
    f = oracle(m)
    x, _ = f.constrained(np.asarray(q, dtype=np.float64))
    tot = 0.0
    for L in m.likelihoods:
        if L.dist != "ordered_probit":
            continue
        y = np.asarray(L.y).astype(int)
        c = np.concatenate([[-np.inf], f.cutpoints(L, x), [np.inf]])
        s, _ = f.scale(L, x)
        eta = f.eta(L, x)[0]
        a, b = (c[y] - eta) / s, (c[y + 1] - eta) / s
        mid = np.isfinite(a) & np.isfinite(b)
        tot += float(np.sum((np.abs(a[mid]) + np.abs(b[mid]) + 1.0) / (b[mid] - a[mid]) ** power))
    return tot


# ------------------------------------------------------------------------------------------------------------------------
# the case catalogue
# ------------------------------------------------------------------------------------------------------------------------
def _case(link, K, cut, eta_kind, sigma, rng, N=16, y_from=None):
    """An ordinal regression with K categories; cut: "var" (ordered variable, Normal(0, 3) prior), "pos" (ordered_positive),
    or an array of constants; eta: "scalar" b0 + b1 x, "indexed" (group effects), "design" (X beta + offsets)."""
    x = rng.standard_normal(N)
    vars_, priors = [], []
    if eta_kind == "scalar":
        vars_ += [Var("b0", "b0", 1), Var("b1", "b1", 1)]
        priors += [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "b1", (0.0, 1.0))]
        terms = [Term([("b0", None)]), Term([("b1", None)], coef=x)]
    elif eta_kind == "indexed":
        vars_ += [Var("a", "a", 4), Var("sa_log__", "sa", 1, "log")]
        priors += [Prior("normal", "a", (0.0, 1.0)), Prior("halfnormal", "sa_log__", (1.0,))]
        terms = [Term([("sa_log__", None), ("a", np.arange(N, dtype=np.int32) % 4)])]
    else:
        vars_ += [Var("beta", "beta", 3)]
        priors += [Prior("normal", "beta", (0.0, 1.0))]
        terms = [Term([("beta", None)], coef=rng.standard_normal((N, 3))), Term([], coef=rng.uniform(-1.0, 1.0, N))]
    if isinstance(cut, str):
        tr = "ordered" if cut == "var" else "ordered_positive"
        z0 = np.concatenate([[-1.0 if cut == "var" else 0.0], np.log(np.full(K - 2, 0.8))])
        vars_.append(Var("c_ordered__", "c", K - 1, tr if K > 2 or cut == "pos" else None, initial=z0[: K - 1]))
        priors.append(Prior("normal", "c_ordered__", (0.0, 3.0)))
        cutpoints = Ref("c_ordered__")
    else:
        cutpoints = np.asarray(cut, dtype=np.float64)
    s = None
    if link == "ordered_probit":
        if sigma == "ref":
            vars_.append(Var("s_log__", "s", 1, "log"))
            priors.append(Prior("halfnormal", "s_log__", (1.5,)))
            s = Ref("s_log__")
        elif sigma == "obs":
            s = rng.uniform(0.5, 1.5, N)
        else:
            s = 0.9
    y = rng.choice(np.arange(K) if y_from is None else np.asarray(y_from), N).astype(np.float64)
    return ModelIR(vars=vars_, priors=priors, likelihoods=[Likelihood(link, y, terms, sigma=s, cutpoints=cutpoints)])


def _tail_case(link, gap):
    """eta_i = b0 + offset_i with offsets out to +-40 around constant cutpoints; gap: the spacing of the middle pair."""
    off = np.array([-40.0, -30.0, -12.0, -3.0, -0.5, 0.0, 0.4, 2.5, 11.0, 25.0, 33.0, 40.0])
    c = np.array([-1.0, 0.0, gap, 1.5])
    y = np.array([0, 4, 2, 2, 1, 2, 3, 0, 4, 2, 1, 3], dtype=np.float64)
    s = 1.0 if link == "ordered_probit" else None
    return ModelIR(vars=[Var("b0", "b0", 1)], priors=[Prior("normal", "b0", (0.0, 3.0))],
                   likelihoods=[Likelihood(link, y, [Term([("b0", None)]), Term([], coef=off)], sigma=s, cutpoints=c)])


CASES = {}
for _l, _sh in (("ordered_logistic", "logit"), ("ordered_probit", "probit")):
    for _K in (2, 3, 5, 7, 8):
        CASES[f"{_sh}-K{_K}-var-scalar"] = (lambda rng, l=_l, K=_K: _case(l, K, "var", "scalar", "const", rng))
    CASES[f"{_sh}-pos-indexed"] = (lambda rng, l=_l: _case(l, 4, "pos", "indexed", "ref", rng))
    CASES[f"{_sh}-const-design"] = (lambda rng, l=_l: _case(l, 5, [-1.5, -0.2, 0.3, 1.8], "design", "obs", rng))
    CASES[f"{_sh}-unobserved"] = (lambda rng, l=_l: _case(l, 6, "var", "design", "ref", rng, y_from=[0, 2, 5]))
    CASES[f"{_sh}-tails"] = (lambda rng, l=_l: _tail_case(l, 0.3))
    CASES[f"{_sh}-narrow"] = (lambda rng, l=_l: _tail_case(l, 1e-6 if l == "ordered_logistic" else 1e-3))
CASE_IDS = list(CASES)


def build(cid):
    return CASES[cid](np.random.default_rng(zlib.crc32(cid.encode())))


def points(m, cid):
    rng = np.random.default_rng(zlib.crc32(cid.encode()) + 1)
    return np.array([m.initial_point() + rng.uniform(-1.0, 1.0, m.n) for _ in range(3)])


@lru_cache(maxsize=None)
def mp_reference(cid):
    m = build(cid)
    Q = points(m, cid)
    lp, S = np.array([_mp_logp(m, q) for q in Q]).T
    return Q, lp, S, np.array([_conditioning(m, q) for q in Q])


def _lp_tol(S, C):
    return LP_TOL * S + 1e-15 * C


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference and the oracle
# ------------------------------------------------------------------------------------------------------------------------
def test_mp_reference_equals_scipy_and_the_reference_known_answers():
    c = [mpf(-2), mpf(0), mpf(2)]
    with mp.workdps(MP_DPS):
        # TestOrderedLogistic / TestOrderedProbit.test_expected_categorical, tests/distributions/test_discrete.py:921-978
        for link, want in (("ordered_logistic", [0.11920292, 0.38079708, 0.38079708, 0.11920292]),
                           ("ordered_probit", [0.02275013, 0.47724987, 0.47724987, 0.02275013])):
            got = [float(mp.exp(_mp_lik(link, y, 4, mpf(0), mpf(1), c))) for y in range(4)]
            np.testing.assert_allclose(got, want, rtol=1e-7)
        cut = np.array([-1.3, -0.1, 0.8, 2.2])
        for eta in (-3.0, -0.4, 0.0, 1.1, 4.0):
            for s in (0.6, 1.0, 1.7):
                cc = np.concatenate([[-np.inf], cut, [np.inf]])
                a, b = cc[:-1] - eta, cc[1:] - eta  # differences of upper tails above the mode: no cancellation
                p_lo = np.where(a > 0, special.expit(-a) - special.expit(-b), special.expit(b) - special.expit(a))
                a, b = a / s, b / s
                p_pr = np.where(a > 0, stats.norm.sf(a) - stats.norm.sf(b), stats.norm.cdf(b) - stats.norm.cdf(a))
                for y in range(5):
                    mc = [mpf(v) for v in cut]
                    lo = float(_mp_lik("ordered_logistic", y, 5, mpf(eta), mpf(1), mc))
                    pr = float(_mp_lik("ordered_probit", y, 5, mpf(eta), mpf(s), mc))
                    assert abs(lo - np.log(p_lo[y])) <= 1e-13 * max(1.0, abs(lo)), (eta, y)
                    assert abs(pr - np.log(p_pr[y])) <= 1e-13 * max(1.0, abs(pr)), (eta, s, y)


def test_the_catalogue_covers_the_ordinal_forms():
    ms = {cid: build(cid) for cid in CASE_IDS}
    links = {m.likelihoods[0].dist for m in ms.values()}
    assert links == set(ir.ORDINAL_LIKS)
    assert {m.likelihoods[0].n_categories(m) for m in ms.values()} >= set(range(2, 9))
    assert any(len(np.unique(m.likelihoods[0].y)) < m.likelihoods[0].n_categories(m) for m in ms.values())
    sig = {type(m.likelihoods[0].sigma).__name__ for m in ms.values() if m.likelihoods[0].dist == "ordered_probit"}
    assert {"Ref", "ndarray", "float"} <= sig
    assert any(ir.is_design(t) for m in ms.values() for t in m.likelihoods[0].terms)
    gaps = [np.min(np.diff(m.likelihoods[0].cutpoints)) for m in ms.values() if not isinstance(m.likelihoods[0].cutpoints, Ref)]
    assert min(gaps) <= 1e-6


@pytest.mark.parametrize("cid", CASE_IDS)
def test_oracle_matches_the_mp_reference_and_central_differences(cid):
    m = build(cid)
    f = oracle(m)
    Q, lp_mp, S, C = mp_reference(cid)
    for q, want, s, c in zip(Q, lp_mp, S, C):
        lp, g = f(q)
        assert abs(lp - want) <= _lp_tol(s, c), (cid, lp, want)
        fd = fd_grad(f, q)
        np.testing.assert_allclose(g, fd, rtol=2e-5, atol=2e-5 * max(1.0, np.max(np.abs(g))), err_msg=cid)


def test_k2_logistic_is_bernoulli_logit_and_probit_is_normal_lcdf():
    rng = np.random.default_rng(3)
    eta = rng.uniform(-30.0, 30.0, 200)
    y = (rng.random(200) < 0.5).astype(float)
    c = 0.7
    from oracle.ir_numpy_ordinal import ordinal_terms

    lp, rs, _, _ = ordinal_terms("ordered_logistic", y, eta, 1.0, [c])
    # y = 1 is the upper category: Bernoulli(logit_p = eta - c) (discrete.py:362-367)
    t = eta - c
    np.testing.assert_allclose(lp, np.where(y == 1, -np.logaddexp(0.0, -t), -np.logaddexp(0.0, t)), rtol=1e-14, atol=1e-300)
    np.testing.assert_allclose(rs, y - special.expit(t), rtol=1e-12, atol=1e-15)
    s = 1.3
    lp, _, _, _ = ordinal_terms("ordered_probit", y, eta, s, [c])
    # normal_lcdf form (dist_math.py:126-142): log Phi((c - eta) / s) for y = 0, log(1 - Phi(...)) for y = 1
    z = (c - eta) / s
    np.testing.assert_allclose(lp, np.where(y == 0, special.log_ndtr(z), special.log_ndtr(-z)), rtol=1e-13)


@pytest.mark.parametrize("size", [1, 2, 33, 300])
@pytest.mark.parametrize("positive", [False, True])
def test_ordered_transform_equals_the_reference_formulas(size, positive):
    rng = np.random.default_rng(size)
    z = rng.normal(0.0, 1.0, (3, size))
    # Ordered.backward / log_jac_det, transforms.py:96-120, restated
    d = np.exp(z) if positive else np.concatenate([z[:, :1], np.exp(z[:, 1:])], axis=1)
    want = np.cumsum(d, axis=-1)
    np.testing.assert_array_equal(ir.ordered_backward(z.copy(), positive), want)
    tr = "ordered_positive" if positive else "ordered"
    m = ModelIR(vars=[Var("c_ordered__", "c", size, tr)], priors=[Prior("normal", "c_ordered__", (0.0, 3.0))])
    np.testing.assert_array_equal(m.constrain(z)["c"] if size > 1 else m.constrain(z)["c"][..., None], want)
    spec = models.ModelSpec(models.KIND_IR, size, models._layout([("c_ordered__", "c", size, tr, None)])[0])
    np.testing.assert_array_equal(np.reshape(spec.constrain(z)["c"], want.shape), want)
    assert np.all(np.diff(want, axis=-1) > 0)
    # the oracle's log|J| and chain rule, against central differences of logp = log|J| + sum_k N(x_k; 0, 3)
    f = oracle(m)
    lp, g = f(z[0])
    jac = np.sum(z[0]) if positive else np.sum(z[0, 1:])
    assert abs(lp - (jac + np.sum(stats.norm.logpdf(want[0], 0.0, 3.0)))) <= 1e-12 * max(1.0, abs(lp))
    np.testing.assert_allclose(g, fd_grad(f, z[0]), rtol=1e-6, atol=1e-6 * max(1.0, np.max(np.abs(g))))


def _ord(link="ordered_logistic", y=(0, 1, 2), cut=Ref("c_ordered__"), tr="ordered", size=2, prior="normal", sigma=None):
    pars = {"normal": (0.0, 1.0), "halfnormal": (1.0,), "uniform": (0.0, 1.0), "exponential": (1.0,)}[prior]
    return ModelIR(vars=[Var("b", "b", 1), Var("c_ordered__", "c", size, tr)],
                   priors=[Prior("normal", "b", (0.0, 1.0)), Prior(prior, "c_ordered__", pars)],
                   likelihoods=[Likelihood(link, np.asarray(y, dtype=float), [Term([("b", None)])], sigma=sigma, cutpoints=cut)])


REFUSALS = [
    ("halfnormal on ordered", dict(prior="halfnormal"), ir.ORDERED_PRIOR),
    ("exponential on ordered", dict(prior="exponential"), ir.ORDERED_PRIOR),
    ("uniform on ordered", dict(prior="uniform"), ir.ORDERED_PRIOR),
    ("uniform on ordered_positive", dict(prior="uniform", tr="ordered_positive"), ir.ORDERED_PRIOR),
    ("y above K - 1", dict(y=(0, 3)), ir.ORD_Y),
    ("negative y", dict(y=(-1, 0)), ir.ORD_Y),
    ("fractional y", dict(y=(0.5, 1)), ir.ORD_Y),
    ("K < 2", dict(cut=np.array([])), ir.ORD_K),
    ("unordered cutpoint variable", dict(tr=None), ir.CUT_ORDERED),
    ("decreasing constants", dict(cut=np.array([0.5, 0.1])), ir.CUT_CONST),
    ("tied constants", dict(cut=np.array([0.5, 0.5])), ir.CUT_CONST),
    ("infinite constants", dict(cut=np.array([-np.inf, 0.5])), ir.CUT_CONST),
    ("sigma on the logistic link", dict(sigma=1.0), ir.LOGISTIC_SIGMA),
    ("probit without sigma", dict(link="ordered_probit"), "needs sigma"),
    ("probit sigma <= 0", dict(link="ordered_probit", sigma=-1.0), "must be a finite constant > 0"),
    ("probit sigma on a real-line variable", dict(link="ordered_probit", sigma=Ref("b")), "must be a finite constant > 0"),
]


@pytest.mark.parametrize("what,kw,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_validate_refuses_each_clause_of_the_support_rule(what, kw, msg):
    with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)").replace("[", r"\[").replace("]", r"\]")):
        _ord(**kw).validate()


def test_validate_accepts_the_allowed_forms_and_refuses_misplaced_cutpoints():
    _ord().validate()
    _ord(tr="ordered_positive", prior="halfnormal").validate()  # ordered_positive is positive support
    _ord(cut=np.array([0.1, 0.4])).validate()
    _ord(size=1, tr=None, y=(0, 1)).validate()  # K = 2: one cutpoint needs no ordering
    m = _ord(link="ordered_probit", sigma=Ref("s_ordered__"))
    m.vars.append(Var("s_ordered__", "s", 1, "ordered_positive"))
    m.validate()  # a size-1 ordered_positive variable is a scale
    bad = ModelIR(vars=[Var("b", "b", 1)], priors=[Prior("normal", "b", (0.0, 1.0))],
                  likelihoods=[Likelihood("normal", np.zeros(3), [Term([("b", None)])], sigma=1.0, cutpoints=np.array([0.0]))])
    with pytest.raises(ValueError, match="cutpoints belong to"):
        bad.validate()


def test_lowered_tables_hold_k_and_the_cutpoint_term():
    m = ir.ordinal_regression_ir("probit", sigma="var")
    low = ir.lower(m)
    L = low.liks[0]
    K = m.likelihoods[0].n_categories(m)
    assert L["dist"] == ir.LIK_DISTS["ordered_probit"] == 11 and L["nu"] == K == 5
    off = m.offsets()["cutpoints_ordered__"]
    assert L["cut"]["coef"] is None and L["cut"]["factors"] == [(off, K - 1, None)]
    assert len(L["terms"]) == 2 and L["sigma_kind"] == ir.SIGMA_REF
    assert low.vars[3][2] == ir.TRANSFORMS["ordered"] == 3 and ir.TRANSFORMS["ordered_positive"] == 4
    assert low.liks[1]["y_var"] == 4  # the cutpoint prior Normal(linspace, 5) is a latent factor
    const = _ord(cut=np.array([-0.5, 0.25]))
    Lc = ir.lower(const).liks[0]
    assert Lc["dist"] == 10 and Lc["nu"] == 3.0 and Lc["cut"]["factors"] == [] and list(Lc["cut"]["coef"]) == [-0.5, 0.25]
    assert np.array_equal(const.constant_data()["y_cutpoints"], [-0.5, 0.25])
    assert ir.specialise(m) is None and ir.specialise(ir.ordinal_regression_ir()) is None
    from pymc_b200 import _lib

    c_ir, keep = _lib.build_ir(low)  # the ctypes table holds the cutpoint term one past the predictor's
    lik = _lib.IrLik.from_address(c_ir.liks)
    assert lik.n_terms == 2
    cut = (_lib.IrTerm * 3).from_address(lik.terms)[2]
    assert cut.n_factors == 1 and cut.f[0].offset == off and cut.f[0].size == K - 1


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
BUILDERS = {
    "logistic": lambda: ir.ordinal_regression_ir("logistic"),
    "probit": lambda: ir.ordinal_regression_ir("probit"),
    "probit_var": lambda: ir.ordinal_regression_ir("probit", sigma="var", seed=5),
    "logistic_k34": lambda: ir.ordinal_regression_ir("logistic", n_obs=900, K=34, seed=6),     # an ordered size of 33
    "probit_k301_cta": lambda: ir.ordinal_regression_ir("probit", n_obs=2000, K=301, seed=7),  # 300: chain = CTA
}


def _device(m):
    from pymc_b200 import engine

    return engine.CompiledModel(m, specialise=False)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", CASE_IDS)
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid):
    m = build(cid)
    cm = _device(m)
    f = oracle(m)
    Q, lp_mp, S, C = mp_reference(cid)
    lo = np.array([f(q)[0] for q in Q])
    go = np.array([f(q)[1] for q in Q])
    C2 = np.array([_conditioning(m, q, 2) for q in Q])
    for team, (lp, g) in logp_at_both_team_shapes(cm, Q).items():
        assert np.all(np.abs(lp - lp_mp) <= _lp_tol(S, C)), (cid, team, lp - lp_mp)
        assert np.all(np.abs(lp - lo) <= _lp_tol(S, C)), (cid, team, lp - lo)
        scale = np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))
        err = np.max(np.abs(g - go) / scale, axis=1)
        assert np.all(err <= 1e-11 + 1e-15 * C2), (cid, team, err, C2)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_device_function_matches_the_oracle_on_the_builders(name):
    m = BUILDERS[name]()
    cm = _device(m)
    assert (m.n > 256) == name.endswith("cta")
    assert not cm.supports_constrain
    f = oracle(m)
    Q = m.initial_point() + np.random.default_rng(0).uniform(-0.5, 0.5, (6, m.n))
    lp, g = cm.logp_dlogp(Q)
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12
    assert np.max(np.abs(g - go) / np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))) <= 1e-11


@pytest.mark.gpu
@pytest.mark.parametrize("name,eps", [("logistic", 0.1), ("probit", 0.1), ("probit_var", 0.1)])
def test_fixed_step_nuts_matches_the_oracle_sampler(name, eps):
    m = BUILDERS[name]()
    fixed_step_against_oracle(m, oracle(m), eps)


@pytest.mark.gpu
@pytest.mark.parametrize("link", ["logistic", "probit"])
def test_lockstep_dense_mass_run_matches_the_oracle(link):
    m = ir.ordinal_regression_ir(link, n_obs=120)
    fixed_step_against_oracle(m, oracle(m), 0.3, dense_cov=random_dense_cov(m.n, 2, 0.02, 0.05, 12), C=2, T=10)


@pytest.mark.gpu
def test_adaptive_run_matches_the_oracle_posterior_and_returns_ordered_cutpoints():
    """64 device chains against 8 oracle chains on the ordinal logistic regression: posterior means within 4 MCSE (an
    effective-size-free bound, SE of the mean of the pooled draws), standard deviations within 25 %; the cutpoint draws of
    sample_b200_nuts come back ordered."""
    import pymc_b200

    m = ir.ordinal_regression_ir("logistic", n_obs=200)
    adaptive_against_oracle(m, oracle(m), chain_seed=23, spread=0.5, philox_seed=5, oracle_seed=200, se_bound=4.0)
    res = pymc_b200.sample_b200_nuts(30, tune=100, chains=4, random_seed=3, model=m, compute_convergence_checks=False)
    c = np.asarray(res.posterior["cutpoints"])
    assert c.shape == (4, 30, 4) and np.all(np.diff(c, axis=-1) > 0)


@pytest.mark.gpu
def test_pointwise_log_likelihood_and_the_log_likelihood_group_match_scipy():
    import pymc_b200

    def scipy_ll(m, q):
        f = oracle(m)
        L = m.likelihoods[0]
        out = np.empty(q.shape[:-1] + (len(L.y),))
        y = np.asarray(L.y).astype(int)
        for ix in np.ndindex(*q.shape[:-1]):
            x, _ = f.constrained(q[ix])
            c = np.concatenate([[-np.inf], f.cutpoints(L, x), [np.inf]])
            eta = f.eta(L, x)[0]
            if L.dist == "ordered_logistic":
                p = special.expit(c[y + 1] - eta) - special.expit(c[y] - eta)
            else:
                s = f.scale(L, x)[0]
                p = stats.norm.cdf((c[y + 1] - eta) / s) - stats.norm.cdf((c[y] - eta) / s)
            out[ix] = np.log(p)
        return out

    for cid in ("logit-K5-var-scalar", "probit-pos-indexed", "probit-const-design", "logit-unobserved"):
        m = build(cid)
        cm = _device(m)
        q = m.initial_point() + np.random.default_rng(4).uniform(-0.5, 0.5, (2, 3, m.n))
        ll = cm.pointwise_loglik(q)
        np.testing.assert_allclose(ll, scipy_ll(m, q), rtol=1e-11, atol=1e-11, err_msg=cid)
    for m in (ir.ordinal_regression_ir("logistic"), ir.ordinal_regression_ir("probit", sigma="var")):
        res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, keep_untransformed=True,
                                         idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
        ll = res.log_likelihood["y"]
        assert ll.shape == (4, 20, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, scipy_ll(m, res.unconstrained), rtol=1e-11, atol=1e-11)


def test_model_create_refuses_malformed_ordinal_tables_through_the_c_abi():
    def set_y(low, v):
        low.liks[0]["y"] = low.liks[0]["y"].copy()
        low.liks[0]["y"][0] = v

    lg = lambda: ir.ordinal_regression_ir("logistic")  # noqa: E731
    pr = lambda: ir.ordinal_regression_ir("probit")  # noqa: E731
    const = lambda: _ord(cut=np.array([-0.5, 0.25]))  # noqa: E731
    cases = [
        (lg, lambda low: set_y(low, 5.0), ir.ORD_Y),
        (lg, lambda low: set_y(low, -1.0), ir.ORD_Y),
        (lg, lambda low: set_y(low, 1.5), ir.ORD_Y),
        (lg, lambda low: low.liks[0].update(nu=1.0), ir.ORD_K),
        (lg, lambda low: low.liks[0].update(nu=6.0), ir.CUT_SIZE),
        (lg, lambda low: low.vars.__setitem__((3, 2), 0), ir.CUT_ORDERED),
        (const, lambda low: low.priors.__setitem__(1, (2, 1, [(0, 1.0, -1)] * 3)), ir.ORDERED_PRIOR),  # HalfNormal
        (const, lambda low: low.liks[0]["cut"].update(coef=np.array([0.3, 0.1])), ir.CUT_CONST),
        (const, lambda low: low.liks[0]["cut"].update(coef=np.array([0.3, np.nan])), ir.CUT_CONST),
        (lg, lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_CONST, sigma_value=1.0), ir.LOGISTIC_SIGMA),
        (pr, lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_CONST, sigma_value=-1.0), "must be a finite constant > 0"),
        (pr, lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_NONE), "needs sigma"),
    ]
    for builder, edit, msg in cases:
        err = refusal_after_edit(builder, edit)
        assert err is not None and msg in err, (msg, err)
