"""Priors whose location is a linear predictor (``ir.Linear``): centred hierarchical models with group-level predictors
and nested groups, evaluated on the generic IR device function as latent factors.

``CASES`` is a small catalogue: both dists (Normal, StudentT); every location term kind (a scalar, an elementwise
vector, an indexed group effect with an empty and with a dominant group, products of 2 and 3 factors, a constant
offset, a design term); every scale kind (a constant, a Ref with a log or an interval transform, one constant per
element); a latent variable that an observed likelihood also reads; two latent factors chained (state -> county ->
observation); and the example model ``ir.radon_centred_ir``.

``_mp_logp`` extends the 40-digit reference of test_ir_closed_set with the latent factors, written from the published
densities (it reads the ModelIR dataclasses only).  The NumPy oracle of latent factors is tests/ir_latent_oracle.py.
CPU: the oracle against the reference and against central differences; what ``validate`` / ``lower`` refuse; the lowered tables of every builder are those of the parent design (y_var = 0);
``specialise`` and ``fuse_design_columns``; ``from_pymc`` on imitation graphs.  GPU: the device function against the
reference and the oracle at chain = warp and chain = CTA; fixed-step NUTS and a lock-step dense-mass run against the
oracle sampler; the centred example against its non-centred twin; the log-likelihood group and the C-ABI refusals."""
import ctypes
import dataclasses
import hashlib
import re
import zlib

import mpmath
import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import stats
from b200_helpers import fd_grad, fixed_step_against_oracle, logp_at_both_team_shapes, random_dense_cov, refusal_after_edit
from test_frontend_mock import fake_pytensor  # noqa: F401
from test_ir_closed_set import (GRAD_TOL, LP_TOL, MP_DPS, SCALE_RULE, _mp_constrain, _mp_factors, _mp_prior_pieces,
                                assert_close_to_reference, points)

import ir_latent_oracle
from pymc_b200 import ir
from pymc_b200.ir import Likelihood, Linear, ModelIR, Prior, Ref, Term, Var


# ------------------------------------------------------------------------------------------------------------------------
# the high-precision reference, with latent factors
# ------------------------------------------------------------------------------------------------------------------------
def _mp_eta(m, terms, N, x):
    eta = [mpf(0)] * N
    for t in terms:
        if ir.is_design(t):
            X, vn = np.asarray(t.coef), m.var(t.factors[0][0]).name
            for i in range(N):
                eta[i] += mp.fsum(mpf(float(X[i, k])) * x[vn][k] for k in range(X.shape[1]))
            continue
        coef = [mpf(1)] * N if t.coef is None else [mpf(float(c)) for c in np.broadcast_to(t.coef, (N,))]
        for i in range(N):
            pr = coef[i]
            for vn, idx in t.factors:
                xv = x[m.var(vn).name]
                pr *= xv[int(idx[i])] if idx is not None else (xv[0] if len(xv) == 1 else xv[i])
            eta[i] += pr
    return eta


def _location_terms(p):
    loc, _ = ir.LINEAR_PRIORS[p.dist]
    a = p.params[loc]
    return a.terms if isinstance(a, Linear) else [Term([(a.var, None)]) if isinstance(a, Ref) else Term([], coef=float(a))]


def _mp_all_factors(m):
    """_mp_factors of the closed set for everything but the latent priors, plus one factor per latent prior."""
    out = _mp_factors(dataclasses.replace(m, priors=[p for p in m.priors if not ir.is_latent(p)]))
    for p in [p for p in m.priors if ir.is_latent(p)]:
        v = m.var(p.var)
        terms = _location_terms(p)
        sc = p.params[ir.LINEAR_PRIORS[p.dist][1]]
        deps = {v.name} | {m.var(vn).name for t in terms for vn, _ in t.factors} | ({m.var(sc.var).name} if isinstance(sc, Ref) else set())

        def f(x, p=p, v=v, terms=terms, sc=sc):
            mu = _mp_eta(m, terms, v.size, x)
            s = [x[m.var(sc.var).name][0]] * v.size if isinstance(sc, Ref) else [mpf(float(c)) for c in np.broadcast_to(sc, (v.size,))]
            lead = [mpf(float(p.params[0]))] if p.dist == "studentt" else []
            return [t for j in range(v.size) for t in _mp_prior_pieces(p.dist, x[v.name][j], lead + [mu[j], s[j]])]
        out.append((deps, f))
    return out


def _mp_logp(m, q):
    with mp.workdps(MP_DPS):
        x, jac = _mp_constrain(m, [mpf(float(t)) for t in q])
        pieces = [t for j in jac for t in j] + [t for _, f in _mp_all_factors(m) for t in f(x)]
        return float(mp.fsum(pieces)), float(mp.fsum(abs(t) for t in pieces))


def _mp_grad(m, q):
    facs, off, g = _mp_all_factors(m), m.offsets(), np.empty(m.n)
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
# the catalogue
# ------------------------------------------------------------------------------------------------------------------------
def _scale(kind, rng, size):
    """(scale parameter, extra vars, extra priors)"""
    if kind == "const":
        return 0.8, [], []
    if kind == "log":
        return Ref("s_log__"), [Var("s_log__", "s", 1, "log")], [Prior("halfnormal", "s_log__", (1.0,))]
    if kind == "int":
        return Ref("w_interval__"), [Var("w_interval__", "w", 1, "interval", (0.1, 3.0))], [Prior("uniform", "w_interval__", (0.1, 3.0))]
    return np.exp(rng.uniform(-0.7, 0.5, size)), [], []


def _latent_case(dist, loc, scale, rng):
    """a[J] ~ dist(location `loc`, scale), observed elementwise by y ~ Normal(a, 0.6) (the latent variable in a likelihood)."""
    J, G = 18, 6
    vars_ = [Var("g0", "g0", 1), Var("g1", "g1", 1)]
    priors = [Prior("normal", "g0", (0.3, 2.0)), Prior("normal", "g1", (0.0, 1.0))]
    u = rng.standard_normal(J)
    if loc == "scalar":
        terms = [Term([("g0", None)])]
    elif loc == "elementwise":  # a vector of the variable's own size, with a scalar coefficient
        vars_.append(Var("e", "e", J))
        priors.append(Prior("normal", "e", (0.0, 0.5)))
        terms = [Term([("e", None)], coef=0.5), Term([("g0", None)])]
    elif loc in ("empty_group", "dominant_group"):
        if loc == "empty_group":  # groups 1 and 4 hold no element
            g = rng.choice([0, 2, 3, 5], J).astype(np.int32)
        else:  # 90 % of the elements in group 2
            g = np.where(rng.random(J) < 0.9, 2, rng.integers(0, G, J)).astype(np.int32)
        vars_.append(Var("r", "r", G))
        priors.append(Prior("normal", "r", (0.0, 1.0)))
        terms = [Term([("g0", None)]), Term([("g1", None)], coef=u), Term([("r", g)])]
    elif loc == "products":  # g1 e_j (2 factors) + 0.5 t r[g_j] g1 (3 factors: a log-scale, an indexed vector, a scalar)
        g = rng.integers(0, G, J).astype(np.int32)
        vars_ += [Var("e", "e", J), Var("r", "r", G), Var("t_log__", "t", 1, "log")]
        priors += [Prior("normal", "e", (0.0, 1.0)), Prior("normal", "r", (0.0, 1.0)), Prior("halfnormal", "t_log__", (1.0,))]
        terms = [Term([("g1", None), ("e", None)]), Term([("t_log__", None), ("r", g), ("g1", None)], coef=0.5)]
    elif loc == "offset_design":  # a constant offset per element + Z @ gamma as one design term
        vars_.append(Var("gamma", "gamma", 3))
        priors.append(Prior("normal", "gamma", (0.0, 1.0)))
        terms = [Term([], coef=0.3 * rng.standard_normal(J)), Term([("gamma", None)], coef=rng.standard_normal((J, 3)))]
    else:  # "ref": a plain scalar location, only the per-element scale makes it latent
        terms = None
    sc, sv, sp = _scale(scale, rng, J)
    vars_ += sv + [Var("a", "a", J)]
    priors += sp
    location = Ref("g0") if terms is None else Linear(terms)
    params = (location, sc) if dist == "normal" else (4.0, location, sc)
    priors.append(Prior(dist, "a", params))
    y = rng.normal(0.5, 1.0, J)
    return ModelIR(vars=vars_, priors=priors, likelihoods=[Likelihood("normal", y, [Term([("a", None)])], sigma=0.6)])


def nested_ir(n_obs=60, n_states=3, n_counties=9, seed=3):
    """Two latent factors chained: state_k ~ Normal(g0 + g1 w_k, 1), county_j ~ Normal(state[state_of_j], sigma_c),
    y_i ~ Normal(county[county_i] + b x_i, sigma_y)."""
    rng = np.random.default_rng(seed)
    w = rng.standard_normal(n_states)
    state_of = (np.arange(n_counties) % n_states).astype(np.int32)
    county = np.concatenate([np.arange(n_counties), rng.integers(0, n_counties, n_obs - n_counties)]).astype(np.int32)
    x = rng.standard_normal(n_obs)
    st = 0.5 + 0.4 * w + 0.3 * rng.standard_normal(n_states)
    ct = st[state_of] + 0.4 * rng.standard_normal(n_counties)
    y = ct[county] + 0.3 * x + 0.5 * rng.standard_normal(n_obs)
    return ModelIR(
        name="nested",
        vars=[Var("g0", "g0", 1), Var("g1", "g1", 1), Var("state", "state", n_states), Var("sigma_c_log__", "sigma_c", 1, "log"),
              Var("county", "county", n_counties), Var("b", "b", 1), Var("sigma_y_log__", "sigma_y", 1, "log")],
        priors=[Prior("normal", "g0", (0.0, 2.0)), Prior("normal", "g1", (0.0, 2.0)),
                Prior("normal", "state", (Linear([Term([("g0", None)]), Term([("g1", None)], coef=w)]), 1.0)),
                Prior("halfnormal", "sigma_c_log__", (1.0,)),
                Prior("normal", "county", (Linear([Term([("state", state_of)])]), Ref("sigma_c_log__"))),
                Prior("normal", "b", (0.0, 1.0)), Prior("halfnormal", "sigma_y_log__", (1.0,))],
        likelihoods=[Likelihood("normal", y, [Term([("county", county)]), Term([("b", None)], coef=x)], sigma=Ref("sigma_y_log__"))])


LATENT_SPECS = [  # (dist, location kind, scale kind)
    ("normal", "scalar", "const"), ("normal", "elementwise", "log"), ("normal", "empty_group", "int"),
    ("normal", "products", "elem"), ("normal", "offset_design", "log"), ("normal", "ref", "elem"),
    ("studentt", "scalar", "log"), ("studentt", "dominant_group", "const"), ("studentt", "products", "int"),
    ("studentt", "offset_design", "elem"), ("studentt", "empty_group", "log"),
]
CASES = {f"{d}-{lk}-{sk}": (lambda rng, s=(d, lk, sk): _latent_case(*s, rng)) for d, lk, sk in LATENT_SPECS}
CASES.update({"nested-state-county-obs": lambda rng: nested_ir(),
              "radon_centred-small": lambda rng: ir.radon_centred_ir(n_obs=50, n_counties=8, n_regions=3, seed=5)})
CASE_IDS = list(CASES)


def build(cid):
    return CASES[cid](np.random.default_rng(zlib.crc32(cid.encode())))


_MP = {}


def mp_reference(cid):
    if cid not in _MP:
        m = build(cid)
        Q = points(m, cid)
        lp, S = np.array([_mp_logp(m, q) for q in Q]).T
        _MP[cid] = Q, lp, S, np.array([_mp_grad(m, q) for q in Q])
    return _MP[cid]


def oracle(m):
    return ir_latent_oracle.make_logp(m)


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference and the oracle
# ------------------------------------------------------------------------------------------------------------------------
def test_mp_latent_factor_equals_scipy():
    m = _latent_case("studentt", "empty_group", "elem", np.random.default_rng(1))
    q = m.initial_point() + np.random.default_rng(2).uniform(-1, 1, m.n)
    x = {k: np.atleast_1d(v) for k, v in m.constrain(q).items()}
    p = m.priors[-1]
    mu = np.zeros(18)
    for t in p.params[1].terms:
        term = np.ones(18) if t.coef is None else np.broadcast_to(t.coef, (18,))
        for vn, idx in t.factors:
            xv = x[m.var(vn).rv_name]
            term = term * (xv[idx] if idx is not None else (xv[0] if len(xv) == 1 else xv))
        mu = mu + term
    want = stats.t.logpdf(x["a"], 4.0, mu, p.params[2]).sum()
    with mp.workdps(MP_DPS):
        xm, _ = _mp_constrain(m, [mpf(float(t)) for t in q])
        got = float(mp.fsum(_mp_all_factors(m)[-1][1](xm)))
    assert abs(got - want) <= 1e-13 * max(1.0, abs(want))


def test_the_catalogue_covers_the_new_ground():
    kinds = set()
    for cid in CASE_IDS:
        m = build(cid)
        m.validate()
        assert m.n <= 64, cid
        lat = [p for p in m.priors if ir.is_latent(p)]
        assert lat, cid
        for p in lat:
            loc, scale = ir.LINEAR_PRIORS[p.dist]
            kinds.add(("dist", p.dist))
            sc = p.params[scale]
            kinds.add(("scale", "ref_" + m.var(sc.var).transform if isinstance(sc, Ref) else ("elem" if np.ndim(sc) else "const")))
            size = m.var(p.var).size
            for t in _location_terms(p):
                if ir.is_design(t):
                    kinds.add(("term", "design"))
                    continue
                kinds.add(("factors", len(t.factors)))
                for vn, idx in t.factors:
                    v = m.var(vn)
                    kinds.add(("term", "indexed" if idx is not None else ("scalar" if v.size == 1 else "elementwise")))
                    if idx is not None:
                        c = np.bincount(idx, minlength=v.size)
                        kinds.add(("empty group", bool(np.any(c == 0))))
                        kinds.add(("dominant group", bool(np.max(c) >= 0.85 * size)))
            used = {m.var(vn).name for L in m.likelihoods for t in L.terms for vn, _ in t.factors}
            kinds.add(("latent in a likelihood", m.var(p.var).name in used))
        names = {m.var(p.var).name for p in lat}
        kinds.add(("chained", any(m.var(vn).name in names for p in lat for t in _location_terms(p) for vn, _ in t.factors)))
    assert {("dist", "normal"), ("dist", "studentt"), ("scale", "const"), ("scale", "ref_log"), ("scale", "ref_interval"),
            ("scale", "elem"), ("term", "scalar"), ("term", "elementwise"), ("term", "indexed"), ("term", "design"),
            ("factors", 0), ("factors", 2), ("factors", 3), ("empty group", True), ("dominant group", True),
            ("latent in a likelihood", True), ("chained", True)} <= kinds


@pytest.mark.parametrize("cid", CASE_IDS)
def test_oracle_matches_the_mp_reference(cid):
    m = build(cid)
    Q, lp_mp, S, g_mp = mp_reference(cid)
    f = oracle(m)
    assert_close_to_reference(np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q]), lp_mp, S, g_mp, cid)


@pytest.mark.parametrize("cid", CASE_IDS)
def test_oracle_gradient_by_central_differences(cid):
    m = build(cid)
    f = oracle(m)
    q = m.initial_point() + np.random.default_rng(7).uniform(-0.8, 0.8, m.n)
    g = f(q)[1]
    fd = fd_grad(f, q, h=1e-5)
    np.testing.assert_allclose(fd, g, rtol=1e-6, atol=1e-6 * max(1.0, np.max(np.abs(g))))


# ------------------------------------------------------------------------------------------------------------------------
# CPU: validation, lowering, routing, fusing
# ------------------------------------------------------------------------------------------------------------------------
def _base(**prior_kw):
    vars_ = [Var("g0", "g0", 1), Var("r", "r", 3), Var("v", "v", 2), Var("s_log__", "s", 1, "log"), Var("a", "a", 5)]
    dist, params = prior_kw.get("prior", ("normal", (Linear([Term([("g0", None)])]), 1.0)))
    return ModelIR(vars=vars_, priors=[Prior(dist, "a", params)])


IDX5 = np.array([0, 1, 2, 1, 0], dtype=np.int32)
MALFORMED = [  # (what, (dist, params), message)
    ("Linear as a normal sigma", ("normal", (0.0, Linear([Term([("s_log__", None)])]))), "prior normal on a: parameter 1 cannot be a Linear"),
    ("Linear as the studentt nu", ("studentt", (Linear([Term([("g0", None)])]), 0.0, 1.0)), "prior studentt on a: parameter 0 cannot be a Linear"),
    ("Linear on a cauchy", ("cauchy", (Linear([Term([("g0", None)])]), 1.0)), "prior cauchy on a: parameter 0 cannot be a Linear"),
    ("Linear on a lognormal", ("lognormal", (Linear([Term([("g0", None)])]), 1.0)), "prior lognormal on a: parameter 0 cannot be a Linear"),
    ("index out of range", ("normal", (Linear([Term([("r", np.array([0, 1, 3, 1, 0]))])]), 1.0)), "prior normal on a: location: index of r out of range"),
    ("index of the wrong length", ("normal", (Linear([Term([("r", IDX5[:4])])]), 1.0)), "prior normal on a: location: the index of r has length 4"),
    ("coef of the wrong length", ("normal", (Linear([Term([("g0", None)], coef=np.ones(4))]), 1.0)), "prior normal on a: location: coef length 4"),
    ("vector of another size", ("normal", (Linear([Term([("v", None)])]), 1.0)), "prior normal on a: location: v (size 2) needs an index"),
    ("design of the wrong shape", ("normal", (Linear([Term([("r", None)], coef=np.ones((4, 3)))]), 1.0)), "prior normal on a: location: X must have shape"),
    ("a vector Ref as the scale", ("normal", (Linear([Term([("g0", None)])]), Ref("r"))), "parameter r must be a scalar variable"),
    ("per-element scale of the wrong length", ("normal", (Linear([Term([("g0", None)])]), np.ones(4))), "sigma per element must be"),
    ("per-element scale with a zero", ("studentt", (3.0, Linear([Term([("g0", None)])]), np.array([1, 1, 0, 1, 1.0]))), "sigma per element must be"),
    ("untransformed Ref as the scale", ("normal", (Linear([Term([("g0", None)])]), Ref("g0"))), SCALE_RULE),
]


@pytest.mark.parametrize("what,prior,msg", MALFORMED, ids=[c[0] for c in MALFORMED])
def test_validate_and_lower_refuse_malformed_locations(what, prior, msg):
    m = _base(prior=prior)
    with pytest.raises(ValueError, match=re.escape(msg)):
        m.validate()
    with pytest.raises(ValueError, match=re.escape(msg)):
        ir.lower(m)


def test_validate_accepts_the_well_formed_locations():
    for prior in [("normal", (Linear([Term([("r", IDX5)]), Term([("v", np.array([0, 1, 1, 0, 0]))], coef=np.arange(5.0))]), Ref("s_log__"))),
                  ("studentt", (5.0, Linear([Term([], coef=np.ones(5)), Term([("r", None)], coef=np.ones((5, 3)))]), np.full(5, 0.5))),
                  ("normal", (0.0, np.full(5, 2.0)))]:
        _base(prior=prior).validate()


def _digest(low):
    """sha256 of every table of a LoweredIR except y_var."""
    h = hashlib.sha256()

    def put(a):
        if a is None:
            h.update(b"none")
            return
        a = np.ascontiguousarray(a)
        h.update(f"{a.dtype.str}{a.shape}".encode() + a.tobytes())

    put(np.int64(low.n))
    put(low.vars)
    put(low.var_bounds)
    for dist, var, pars in low.priors:
        put(np.array([dist, var], dtype=np.int64))
        for kind, value, ref in pars:
            put(np.array([kind, ref], dtype=np.int64))
            put(np.float64(value))
    for L in low.liks:
        put(np.array([L["dist"], L["N"], L["sigma_kind"], L["sigma_ref"]], dtype=np.int64))
        put(np.array([L["sigma_value"], L["nu"]], dtype=np.float64))
        put(L["y"])
        put(L["sigma_obs"])
        for T in L["terms"]:
            put(T["coef"])
            put(np.int64(T.get("n_cols", 0)))
            for o, sz, idx in T["factors"]:
                put(np.array([o, sz], dtype=np.int64))
                put(idx)
    for var, phi, sigma, init in low.ar1:
        put(np.array([var, phi[0], phi[2], sigma[0], sigma[2]], dtype=np.int64))
        put(np.array([phi[1], sigma[1], init], dtype=np.float64))
    return h.hexdigest()[:16]


# digests of the lowered tables of every builder, taken before the latent factors existed
PARENT_DIGESTS = {
    "eight_schools_ir": "09aab60d1dca5b53",
    "radon_ir": "32022096d9697450",
    "stochvol_ir": "886bbbb48944cf53",
    "varying_intercept_logistic_ir": "1fac5899e40b3e50",
    "binomial_logit_ir": "1003bdc1a89438f5",
    "negative_binomial_ir": "6680700f3b82c171",
    "gamma_regression_ir": "c3b2c6ef4a51221a",
}


@pytest.mark.parametrize("builder", list(PARENT_DIGESTS))
def test_every_builder_lowers_to_the_tables_it_had(builder):
    from pymc_b200 import _lib

    m = getattr(ir, builder)()
    low = ir.lower(m)
    assert _digest(low) == PARENT_DIGESTS[builder]
    assert len(low.liks) == len(m.likelihoods) and all(L["y_var"] == 0 for L in low.liks)
    c_ir, keep = _lib.build_ir(low)
    assert all(ctypes.cast(c_ir.liks, ctypes.POINTER(_lib.IrLik))[k].y_var == 0 for k in range(c_ir.n_liks))


def test_latent_factors_lower_after_the_observed_likelihoods():
    from pymc_b200 import _lib

    m = nested_ir()
    low = ir.lower(m)
    idx = {v.name: k for k, v in enumerate(m.vars)}
    off = m.offsets()
    assert len(low.priors) == 5 and len(low.liks) == 3  # the two latent priors left the prior table
    assert low.liks[0]["y_var"] == 0 and low.liks[0]["N"] == len(m.likelihoods[0].y)
    st, ct = low.liks[1], low.liks[2]
    assert (st["y_var"], st["N"], st["y"], st["dist"]) == (idx["state"] + 1, 3, None, ir.LIK_DISTS["normal"])
    assert (st["sigma_kind"], st["sigma_value"]) == (ir.SIGMA_CONST, 1.0)
    assert (ct["y_var"], ct["N"], ct["sigma_kind"], ct["sigma_ref"]) == (idx["county"] + 1, 9, ir.SIGMA_REF, off["sigma_c_log__"])
    assert ct["terms"][0]["factors"][0][:2] == (off["state"], 3)
    c_ir, keep = _lib.build_ir(low)
    liks = ctypes.cast(c_ir.liks, ctypes.POINTER(_lib.IrLik))
    assert [liks[k].y_var for k in range(3)] == [0, idx["state"] + 1, idx["county"] + 1] and not liks[1].y
    # a StudentT latent factor carries nu; one constant scale per element goes to sigma_obs
    low = ir.lower(_latent_case("studentt", "offset_design", "elem", np.random.default_rng(0)))
    L = low.liks[-1]
    assert L["dist"] == ir.LIK_DISTS["studentt"] and L["nu"] == 4.0 and L["sigma_kind"] == ir.SIGMA_OBS and len(L["sigma_obs"]) == 18
    assert L["terms"][1]["n_cols"] == 3


def test_host_side_groups_see_no_latent_factor():
    m = ir.radon_centred_ir()
    assert list(m.observed_data()) == ["y"]
    assert set(m.constant_data()) == {"y_coef1", "y_a_idx"}
    draws = m.constrain(np.tile(m.initial_point(), (2, 3, 1)))
    assert draws["a"].shape == (2, 3, 32) and m.eval_deterministics(draws) == {}


def test_specialise_skips_latent_models_and_routes_the_hand_kernels():
    assert ir.specialise(ir.radon_centred_ir()) is None and ir.specialise(nested_ir()) is None
    assert ir.specialise(_base(prior=("normal", (0.0, np.full(5, 2.0))))) is None
    assert ir.specialise(ir.radon_ir()) is not None and ir.specialise(ir.eight_schools_ir()) is not None


def test_fuse_design_columns_fuses_a_run_inside_a_linear_location():
    rng = np.random.default_rng(4)
    J, K = 12, 3
    Z = rng.standard_normal((J, K))
    cols = [Term([("gamma", np.full(J, k, dtype=np.int32))], coef=Z[:, k].copy()) for k in range(K)]
    m = ModelIR(vars=[Var("gamma", "gamma", K), Var("g0", "g0", 1), Var("s_log__", "s", 1, "log"), Var("a", "a", J)],
                priors=[Prior("normal", "gamma", (0.0, 1.0)), Prior("normal", "g0", (0.0, 1.0)), Prior("halfnormal", "s_log__", (1.0,)),
                        Prior("normal", "a", (Linear([Term([("g0", None)])] + cols), Ref("s_log__")))],
                likelihoods=[Likelihood("normal", rng.standard_normal(J), [Term([("a", None)])], sigma=0.5)])
    f = ir.fuse_design_columns(m)
    T = f.priors[-1].params[0].terms
    assert len(T) == 2 and T[0].factors == [("g0", None)] and ir.is_design(T[1]) and np.array_equal(T[1].coef, Z)
    assert len(m.priors[-1].params[0].terms) == 4  # the model itself is not changed
    fo, fm = oracle(f), oracle(m)
    for q in m.initial_point() + rng.uniform(-1, 1, (4, m.n)):
        (a, ga), (b, gb) = fo(q), fm(q)
        assert abs(a - b) <= 1e-13 * abs(b)
        np.testing.assert_allclose(ga, gb, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------------
# CPU: from_pymc on imitation graphs
# ------------------------------------------------------------------------------------------------------------------------
def _hand_density(m, fn):
    """fn(x: rv name -> constrained values) -> log p without Jacobians; compared with the oracle at random points."""
    f = oracle(m)
    rng = np.random.default_rng(0)
    for _ in range(4):
        q = m.initial_point() + rng.uniform(-0.7, 0.7, m.n)
        x = {k: np.atleast_1d(v) for k, v in m.constrain(q).items()}
        jac = sum(q[m.offsets()[v.name]: m.offsets()[v.name] + v.size].sum() for v in m.vars if v.transform == "log")
        assert abs(f(q)[0] - (fn(x) + jac)) <= 1e-11 * max(1.0, abs(f(q)[0]))


def _radon_graph(form):
    from test_frontend_mock import AdvancedSubtensor1, Constant, FakeModel, LogTransform, apply, bcast, elem, rv

    rng = np.random.default_rng(11)
    J, S, N = 6, 2, 30
    u, state_of = rng.standard_normal(J), np.array([0, 1, 0, 1, 1, 0])
    county = rng.integers(0, J, N)
    y = rng.standard_normal(N)
    M = FakeModel(form)
    g0 = M.free(rv("NormalRV", "g0", Constant(0.0), Constant(5.0)), 1)
    g1 = M.free(rv("NormalRV", "g1", Constant(0.0), Constant(5.0)), 1)
    sa = M.free(rv("HalfNormalRV", "sigma_a", Constant(0.0), Constant(1.0)), 1, LogTransform())
    if form == "nested":
        st = M.free(rv("NormalRV", "a_state", elem("Add", bcast(g0), elem("Mul", bcast(g1), Constant(np.array([0.5, -1.0])))),
                       Constant(1.0)), S)
        loc = apply(AdvancedSubtensor1(), st, Constant(state_of))
    else:
        loc = elem("Add", bcast(g0), elem("Mul", bcast(g1), Constant(u)))
        if form == "deterministic":
            loc = elem("Identity", loc)  # pm.Deterministic("mu_a", ...): a named copy of the expression
    a = M.free(rv("NormalRV", "a", loc, bcast(sa)), J)
    M.observe(rv("NormalRV", "y", apply(AdvancedSubtensor1(), a, Constant(county)), Constant(np.full(N, 0.7))), y)
    data = dict(u=u, state_of=state_of, county=county, y=y)
    return M, data


@pytest.mark.parametrize("form", ["predictor", "nested", "deterministic"])
def test_from_pymc_lowers_group_level_locations(fake_pytensor, form):
    from pymc_b200 import from_pymc

    M, d = _radon_graph(form)
    m = from_pymc(M)
    assert isinstance(m.priors[-1].params[0], Linear) and ir.is_latent(m.priors[-1])

    def density(x):
        n = stats.norm.logpdf
        lp = n(x["g0"], 0, 5).sum() + n(x["g1"], 0, 5).sum() + stats.halfnorm.logpdf(x["sigma_a"], scale=1.0).sum()
        if form == "nested":
            lp += n(x["a_state"], x["g0"] + x["g1"] * np.array([0.5, -1.0]), 1.0).sum()
            mu = x["a_state"][d["state_of"]]
        else:
            mu = x["g0"] + x["g1"] * d["u"]
        return lp + n(x["a"], mu, x["sigma_a"]).sum() + n(d["y"], x["a"][d["county"]], 0.7).sum()
    _hand_density(m, density)


def test_from_pymc_sees_through_a_deterministic_in_a_likelihood_location(fake_pytensor):
    from test_frontend_mock import Constant, FakeModel, bcast, elem, rv

    from pymc_b200 import from_pymc

    M = FakeModel("det")
    b = M.free(rv("NormalRV", "b", Constant(0.0), Constant(1.0)), 1)
    x = np.array([0.5, 1.0, -2.0])
    M.observe(rv("NormalRV", "y", elem("Identity", elem("Mul", bcast(b), Constant(x))), Constant(1.0)), np.zeros(3))
    m = from_pymc(M)
    _hand_density(m, lambda v: stats.norm.logpdf(v["b"], 0, 1).sum() + stats.norm.logpdf(np.zeros(3), v["b"] * x, 1.0).sum())


def test_from_pymc_takes_a_constant_vector_sigma(fake_pytensor):
    from test_frontend_mock import Constant, FakeModel, rv

    from pymc_b200 import from_pymc

    s = np.array([0.5, 1.0, 2.0])
    M = FakeModel("vsig")
    M.free(rv("NormalRV", "a", Constant(0.3), Constant(s)), 3)
    m = from_pymc(M)
    assert np.array_equal(m.priors[0].params[1], s) and ir.is_latent(m.priors[0])
    _hand_density(m, lambda v: stats.norm.logpdf(v["a"], 0.3, s).sum())


def test_from_pymc_refuses_the_out_of_scope_forms(fake_pytensor):
    from test_frontend_mock import AdvancedSubtensor1, Constant, FakeModel, LogTransform, apply, bcast, elem, rv

    from pymc_b200 import from_pymc

    def model(kind):
        M = FakeModel(kind)
        g0 = M.free(rv("NormalRV", "g0", Constant(0.0), Constant(1.0)), 1)
        sg = M.free(rv("HalfNormalRV", "sg", Constant(0.0), Constant(1.0)), 2, LogTransform())
        loc = elem("Add", bcast(g0), Constant(np.arange(4.0)))
        if kind == "halfnormal":
            M.free(rv("HalfNormalRV", "h", loc, Constant(1.0)), 4, LogTransform())
        elif kind == "lognormal":
            M.free(rv("LogNormalRV", "h", loc, Constant(1.0)), 4, LogTransform())
        elif kind == "indexed_sigma":
            M.free(rv("NormalRV", "h", loc, apply(AdvancedSubtensor1(), sg, Constant(np.array([0, 1, 0, 1])))), 4)
        else:  # a vector free RV as sigma
            M.free(rv("NormalRV", "h", bcast(g0), sg), 2)
        return M
    for kind, msg in [("halfnormal", "h: halfnormal with a non-zero location"),
                      ("lognormal", "h.param0: parameter is neither a constant scalar nor a scalar free RV"),
                      ("indexed_sigma", "h.param1: parameter is neither a constant scalar nor a scalar free RV"),
                      ("vector_sigma", "h.param1: a vector random variable as a distribution parameter")]:
        with pytest.raises(NotImplementedError, match=re.escape(msg)):
            from_pymc(model(kind))


def test_real_pymc_centred_models_lower_to_their_own_density():
    pm = pytest.importorskip("pymc")
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(0)
    J, N = 6, 40
    u, region, county = rng.standard_normal(J), np.array([0, 1, 2, 0, 1, 2]), rng.integers(0, J, N)
    y = rng.standard_normal(N)
    with pm.Model() as model:
        g0, g1 = pm.Normal("g0", 0, 5), pm.Normal("g1", 0, 5)
        r = pm.Normal("r", 0, 1, shape=3)
        sigma_a = pm.HalfNormal("sigma_a", 1)
        mu_a = pm.Deterministic("mu_a", g0 + g1 * u + r[region])
        a = pm.Normal("a", mu=mu_a, sigma=sigma_a, shape=J)
        pm.Normal("y", a[county], 0.7, observed=y)
    m = from_pymc(model)
    assert ir.is_latent(m.priors[-1])
    f, g = model.logp_dlogp_function(ravel_inputs=True), oracle(m)
    f.set_extra_values({})
    for q in m.initial_point() + np.random.default_rng(1).uniform(-0.5, 0.5, (3, m.n)):
        (lp_ref, dlp_ref), (lp, dlp) = f(q), g(q)
        np.testing.assert_allclose(lp, lp_ref, rtol=1e-9)
        np.testing.assert_allclose(dlp, dlp_ref, rtol=1e-7, atol=1e-9)


# ------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cid", CASE_IDS)
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid):
    from pymc_b200 import engine

    m = build(cid)
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = oracle(m)
    Q, lp_mp, S, g_mp = mp_reference(cid)
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    out = logp_at_both_team_shapes(cm, Q)
    for team, (lp, g) in out.items():
        assert_close_to_reference(lp, g, lp_mp, S, g_mp, (cid, team))
        assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12, (cid, team)
        assert np.max(np.abs(g - go) / np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))) <= 1e-12, (cid, team)
    (lw, gw), (lc, gc) = out["warp"], out["cta"]
    assert np.all(np.abs(lw - lc) <= LP_TOL * S), cid
    assert np.all(np.max(np.abs(gw - gc), axis=1) <= GRAD_TOL * np.maximum(1.0, np.max(np.abs(gw), axis=1))), cid


@pytest.mark.gpu
@pytest.mark.parametrize("team", ["warp", "cta"])
@pytest.mark.parametrize("name,eps", [("radon_centred", 0.05), ("nested", 0.1)])
def test_fixed_step_nuts_matches_the_oracle_sampler(name, eps, team, monkeypatch):
    if team == "cta":
        monkeypatch.setenv("B200_FORCE_TEAM", "1")
    m = ir.radon_centred_ir() if name == "radon_centred" else nested_ir()
    fixed_step_against_oracle(m, oracle(m), eps, C=2, T=10)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle_on_the_example():
    m = ir.radon_centred_ir()
    fixed_step_against_oracle(m, oracle(m), 0.3, dense_cov=random_dense_cov(m.n, 3, 0.01, 0.03, 6), C=2, T=10)


def radon_noncentred_ir(**kw):
    """The example model written with today's terms: a[county] = g0 + g1 u[county] + r[region[county]] + sigma_a z[county]."""
    c = ir.radon_centred_ir(**kw)
    loc = c.priors[4].params[0].terms
    u, region = loc[1].coef, loc[2].factors[0][1]
    L = c.likelihoods[0]
    county, floor = L.terms[0].factors[0][1], L.terms[1].coef
    vars_ = [v if v.name != "a" else Var("z", "z", v.size) for v in c.vars]
    priors = [p if p.var != "a" else Prior("normal", "z", (0.0, 1.0)) for p in c.priors]
    terms = [Term([("g0", None)]), Term([("g1", None)], coef=u[county]), Term([("r", region[county])]),
             Term([("sigma_a_log__", None), ("z", county)]), Term([("b", None)], coef=floor)]
    return ModelIR(name="radon_noncentred", vars=vars_, priors=priors,
                   likelihoods=[Likelihood("normal", L.y, terms, sigma=Ref("sigma_y_log__"))])


@pytest.mark.gpu
def test_centred_and_non_centred_examples_agree():
    """Adaptive NUTS on the centred example and on its non-centred twin: the posterior means of g0, g1, sigma_a, b and
    sigma_y agree within 4 MCSE (MCSE = sd / sqrt(bulk ESS) of each run)."""
    from pymc_b200 import engine
    from pymc_b200 import rng as brng
    from pymc_b200.diagnostics import ess_bulk

    out = {}
    for m in (ir.radon_centred_ir(), radon_noncentred_ir()):
        cm = engine.CompiledModel(m)
        assert cm.spec.name == "ir"
        C = 32
        sr, _, js = brng.chain_generators(17, C)
        q0 = np.stack([m.initial_point() + np.random.default_rng(s).uniform(-1, 1, m.n) for s in js])
        run = cm.nuts_run(q0, brng.pack_pcg64(sr), tune=600, draws=500, mean0=np.broadcast_to(q0.mean(0), q0.shape).copy(),
                          store_warmup=False, philox_seed=5)
        assert run.stats["diverging"].mean() < 0.01, m.name
        x = m.constrain(run.draws)
        out[m.name] = {k: (x[k].mean(), x[k].std() / np.sqrt(ess_bulk(x[k])[0])) for k in ("g0", "g1", "sigma_a", "b", "sigma_y")}
    c, nc = out["radon_centred"], out["radon_noncentred"]
    for k in c:
        assert abs(c[k][0] - nc[k][0]) <= 4.0 * np.hypot(c[k][1], nc[k][1]), (k, c[k], nc[k])


@pytest.mark.gpu
def test_log_likelihood_group_holds_only_the_observed_likelihood():
    import pymc_b200
    from pymc_b200 import _lib, engine

    m = ir.radon_centred_ir()
    res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, keep_untransformed=True,
                                     idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
    assert list(res.log_likelihood) == ["y"]
    L = m.likelihoods[0]
    county, floor = L.terms[0].factors[0][1], L.terms[1].coef
    a, b, sy = res.posterior["a"], res.posterior["b"], res.posterior["sigma_y"]
    want = stats.norm.logpdf(L.y, a[..., county] + b[..., None] * floor, sy[..., None])
    np.testing.assert_allclose(res.log_likelihood["y"], want, rtol=1e-12, atol=1e-12)
    # the latent factor (lowered index 1) is not a likelihood: the C ABI refuses it
    cm = engine.CompiledModel(m, specialise=False)
    lib = _lib.load()
    q = np.ascontiguousarray(np.tile(m.initial_point(), (2, 1)))
    out = np.empty((2, 64))
    assert lib.b200_pointwise_loglik(cm._h, 1, q.ctypes.data, 2, out.ctypes.data, _lib.MEM_HOST, None) != 0
    assert "latent factor" in lib.b200_last_error().decode()
    assert lib.b200_pointwise_loglik(cm._h, 0, q.ctypes.data, 2, np.empty((2, len(L.y))).ctypes.data, _lib.MEM_HOST, None) == 0


def test_model_create_refuses_malformed_latent_tables():
    def setter(**kw):
        return lambda low: low.liks[2].update(kw)

    n_vars = len(nested_ir().vars)
    for edit, msg in [(setter(y_var=-1), "outside [0, n_vars"), (setter(y_var=n_vars + 1), "outside [0, n_vars"),
                      (setter(dist=ir.LIK_DISTS["poisson_log"]), "a latent factor (y_var > 0) is a normal or studentt prior"),
                      (setter(y_var=1), "must equal the size of its variable"),
                      (setter(y_var=0), "missing observations"),
                      (setter(sigma_kind=ir.SIGMA_CONST, sigma_value=-1.0), "sigma must be a finite constant > 0")]:
        err = refusal_after_edit(nested_ir, edit)
        assert err is not None and msg in err, (msg, err)
