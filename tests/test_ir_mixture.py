"""Finite mixtures for IR models: the simplex transform, the Dirichlet prior, and the normal_mixture / poisson_mixture
likelihoods on the generic device function.

``_mp_logp`` writes the joint log-density with mpmath at 40 digits from the published definitions: w = softmax([z, -sum z])
with log|J| = log K + sum log w (SimplexTransform, transforms.py:1091-1116), the Dirichlet (multivariate.py:557-585) and
logsumexp_k(log w_k + log f_k(y_i)) (mixture_logprob, mixture.py:469-494); the gradient is ``mpmath.diff``.  Its pieces
are checked against scipy.stats, the log-Jacobian against slogdet of a finite-difference Jacobian of w_1..w_{K-1}.  The
NumPy oracle (oracle/ir_numpy_mixture.py) is checked against it and central differences, and the device against both."""
import copy
import dataclasses

import mpmath
import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import stats
from scipy.special import logsumexp
from b200_helpers import (adaptive_against_oracle, create_raw, fd_grad, fixed_step_against_oracle, logp_at_both_team_shapes,
                          random_dense_cov, refusal_after_edit)

from pymc_b200 import ir
from pymc_b200.ir import Likelihood, ModelIR, Prior, Ref, Term, Var

MP_DPS = 40


# ------------------------------------------------------------------------------------------------------------------------
# the 40-digit reference
# ------------------------------------------------------------------------------------------------------------------------
def _mp_simplex(z):
    """(log w as mpf, log|J|) of a simplex variable's unconstrained z."""
    ze = [mpf(v) for v in z] + [-mp.fsum(mpf(v) for v in z)]
    lse = mp.log(mp.fsum(mp.exp(v) for v in ze))
    lw = [v - lse for v in ze]
    return lw, mp.log(len(ze)) + mp.fsum(lw)


def _mp_dirichlet(lw, a):
    K = len(lw)
    a = [mpf(v) for v in np.broadcast_to(np.asarray(a, dtype=np.float64), (K,))]
    return mp.loggamma(mp.fsum(a)) - mp.fsum(mp.loggamma(v) for v in a) + mp.fsum((a[k] - 1) * lw[k] for k in range(K))


def _mp_mixture(dist, y, eta, lw, c, s):
    """log p(y) of one observation with every constant; a -inf log weight drops its component."""
    terms = []
    for k in range(len(lw)):
        if lw[k] == -mp.inf:
            continue
        if dist == "normal_mixture":
            z = (mpf(y) - eta - c[k]) / s[k]
            lf = -z * z / 2 - mp.log(s[k]) - mp.log(2 * mp.pi) / 2
        else:
            mu = c[k] * mp.exp(eta)
            lf = mpf(y) * mp.log(mu) - mu - mp.loggamma(mpf(y) + 1)
        terms.append(lw[k] + lf)
    m = max(terms)
    return m + mp.log(mp.fsum(mp.exp(t - m) for t in terms))


def _mp_constrain(m, q):
    """name -> constrained values (mpf lists; a simplex variable: its log weights) and the sum of the log-Jacobians."""
    off, x, lj = m.offsets(), {}, mpf(0)
    for v in m.vars:
        z = list(q[off[v.name]:off[v.name] + v.size])
        if v.transform == "log":
            x[v.name], lj = [mp.exp(t) for t in z], lj + mp.fsum(z)
        elif v.transform in ("ordered", "ordered_positive"):
            pos = v.transform == "ordered_positive"
            acc, vals = (mp.exp(z[0]) if pos else z[0]), []
            vals.append(acc)
            for t in z[1:]:
                acc = acc + mp.exp(t)
                vals.append(acc)
            x[v.name], lj = vals, lj + mp.fsum(z if pos else z[1:])
        elif v.transform == "simplex":
            x[v.name], l = _mp_simplex(z)
            lj += l
        else:
            x[v.name] = z
    return x, lj


def _mp_parts(m, qq):
    """Every part of the joint log-density, with its constants, at mpf coordinates qq."""
    x, lj = _mp_constrain(m, qq)
    parts = [lj]
    for p in m.priors:
        xv = x[m.var(p.var).name]
        if p.dist == "dirichlet":
            parts.append(_mp_dirichlet(xv, p.params[0]))
        elif p.dist == "normal":
            mu, s = mpf(p.params[0]), mpf(p.params[1])
            parts += [-((t - mu) / s) ** 2 / 2 - mp.log(s) - mp.log(2 * mp.pi) / 2 for t in xv]
        elif p.dist == "halfnormal":
            s = mpf(p.params[0])
            parts += [-(t / s) ** 2 / 2 - mp.log(s) + mp.log(2 / mp.pi) / 2 for t in xv]
        else:
            raise NotImplementedError(p.dist)
    for L in m.likelihoods:
        K = L.n_components(m)

        def blk(a):
            return x[m.var(a.var).name] if isinstance(a, Ref) else [mpf(float(v)) for v in np.broadcast_to(a, (K,))]

        lw = x[m.var(L.weights.var).name] if isinstance(L.weights, Ref) else \
            [mp.log(mpf(float(w))) if w > 0 else -mp.inf for w in L.weights]
        c = blk(L.components)
        s = None
        if L.dist == "normal_mixture":
            s = blk(L.sigma)
            s = s * K if len(s) == 1 else s
        for i, y in enumerate(L.y):
            eta = mpf(0)
            for t in L.terms:
                if ir.is_design(t):
                    b = x[m.var(t.factors[0][0]).name]
                    eta += mp.fsum(mpf(float(t.coef[i, k])) * b[k] for k in range(len(b)))
                else:
                    eta += x[m.var(t.factors[0][0]).name][0]
            parts.append(_mp_mixture(L.dist, y, eta, lw, c, s))
    return parts


def _mp_logp(m, q):
    """(logp, the sum of the magnitudes of its parts)."""
    with mp.workdps(MP_DPS):
        parts = _mp_parts(m, [mpf(float(v)) for v in q])
        return float(mp.fsum(parts)), float(mp.fsum(abs(p) for p in parts))


def _mp_grad(m, q):
    with mp.workdps(MP_DPS):
        q0 = [mpf(float(v)) for v in q]
        g = np.empty(len(q))
        for j in range(len(q)):
            def h(t, j=j):
                qq = list(q0)
                qq[j] = t
                return mp.fsum(_mp_parts(m, qq))
            g[j] = float(mpmath.diff(h, q0[j]))
        return g


# ------------------------------------------------------------------------------------------------------------------------
# the catalogue: K = 2, 3, 5; every weights / components / sigma kind; with and without eta; a zero constant weight; a
# component whose responsibility underflows; log w_k near -700
# ------------------------------------------------------------------------------------------------------------------------
def _model(dist, K, weights, comp, sigma=None, eta=None, y=None, N=12, seed=0):
    rng = np.random.default_rng(seed)
    vars_, priors, terms = [], [], []
    if isinstance(weights, str):
        vars_.append(Var("w_simplex__", "w", K - 1, "simplex"))
        priors.append(Prior("dirichlet", "w_simplex__", (np.full(K, 1.5),)))
        wt = Ref("w_simplex__")
    else:
        wt = np.asarray(weights, dtype=np.float64)
    if isinstance(comp, str):  # "ordered", "none", "ordered_positive", "log"
        vars_.append(Var("c", "c", K, None if comp == "none" else comp,
                         initial=np.concatenate([[-1.0 if comp in ("ordered", "none") else 0.0], np.zeros(K - 1)])))
        priors.append(Prior("normal", "c", (0.0, 5.0)))
        ct = Ref("c")
    else:
        ct = np.asarray(comp, dtype=np.float64)
    if isinstance(sigma, int):  # a variable of that size
        vars_.append(Var("s_log__", "s", sigma, "log"))
        priors.append(Prior("halfnormal", "s_log__", (2.0,)))
        sigma = Ref("s_log__")
    if eta == "design":
        vars_.append(Var("beta", "beta", 2))
        priors.append(Prior("normal", "beta", (0.0, 1.0)))
        terms = [Term([("beta", None)], coef=rng.standard_normal((N, 2)))]
    elif eta == "scalar":
        vars_.append(Var("b0", "b0", 1))
        priors.append(Prior("normal", "b0", (0.0, 1.0)))
        terms = [Term([("b0", None)])]
    if y is None:
        y = rng.normal(0.0, 2.0, N) if dist == "normal_mixture" else rng.poisson(3.0, N).astype(np.float64)
    return ModelIR(vars=vars_, priors=priors, name=f"{dist}_{K}",
                   likelihoods=[Likelihood(dist, np.asarray(y, dtype=np.float64), terms, sigma=sigma, weights=wt, components=ct)])


CASES = {
    "normal_k2_simplex_ordered_scalar_sigma": lambda: _model("normal_mixture", 2, "var", "ordered", 1),
    "normal_k3_simplex_ordered_vector_sigma_design": lambda: _model("normal_mixture", 3, "var", "ordered", 3, "design"),
    "normal_k5_const_w_free_mu_const_sigmas": lambda: _model("normal_mixture", 5, np.full(5, 0.2), "none",
                                                             np.linspace(0.5, 2.0, 5)),
    "normal_k3_zero_weight_const_mu_const_sigma_eta": lambda: _model("normal_mixture", 3, [0.5, 0.0, 0.5], [-2.0, 0.0, 2.0],
                                                                     1.3, "scalar"),
    "normal_k3_underflowing_component": lambda: _model("normal_mixture", 3, "var", [0.0, 1.0, 40.0], 1.0,
                                                       y=np.linspace(-1.0, 1.5, 10)),
    "normal_k3_log_w_near_minus_700": lambda: _model("normal_mixture", 3, "var", "ordered", 1),
    "poisson_k2_simplex_ordered_positive": lambda: _model("poisson_mixture", 2, "var", "ordered_positive"),
    "poisson_k3_const_w_const_lam_design": lambda: _model("poisson_mixture", 3, [0.2, 0.3, 0.5], [0.5, 3.0, 9.0], None,
                                                          "design"),
    "poisson_k5_simplex_log_lam_eta": lambda: _model("poisson_mixture", 5, "var", "log", None, "scalar"),
}


def _points(cid, m):
    Q = m.initial_point() + np.random.default_rng(len(cid)).uniform(-0.5, 0.5, (3, m.n))
    if cid == "normal_k3_log_w_near_minus_700":
        Q[:, 0:2] = [350.0, 0.0]  # z~ = (350, 0, -350): log w = (0, -350, -700)
    return Q


def test_the_catalogue_covers_the_mixture_forms():
    ms = [f() for f in CASES.values()]
    Ks = {L.n_components(m) for m in ms for L in m.likelihoods}
    assert Ks == {2, 3, 5}
    Ls = [(m, m.likelihoods[0]) for m in ms]
    assert {L.dist for _, L in Ls} == set(ir.MIXTURE_LIKS)
    assert any(isinstance(L.weights, Ref) for _, L in Ls) and any(not isinstance(L.weights, Ref) for _, L in Ls)
    assert any(not isinstance(L.weights, Ref) and np.any(np.asarray(L.weights) == 0) for _, L in Ls)
    comp = {"const" if not isinstance(L.components, Ref) else m.var(L.components.var).transform or "none" for m, L in Ls}
    assert comp >= {"const", "none", "ordered", "ordered_positive", "log"}
    sig = {("var", m.var(L.sigma.var).size > 1) if isinstance(L.sigma, Ref) else ("const", np.ndim(L.sigma) == 1)
           for m, L in Ls if L.dist == "normal_mixture"}
    assert sig == {("var", False), ("var", True), ("const", False), ("const", True)}
    assert any(L.terms for _, L in Ls) and any(not L.terms for _, L in Ls)
    assert "normal_k3_underflowing_component" in CASES and "normal_k3_log_w_near_minus_700" in CASES


def test_mp_pieces_equal_scipy():
    """The Dirichlet, both mixture densities and the simplex log-Jacobian, against scipy and a finite-difference slogdet."""
    rng = np.random.default_rng(3)
    with mp.workdps(MP_DPS):
        for K in (2, 3, 5):
            z = rng.normal(0.0, 1.0, K - 1)
            lw, lj = _mp_simplex(z)
            w = np.array([float(mp.exp(v)) for v in lw])
            np.testing.assert_allclose(w, ir.simplex_backward(z), rtol=1e-14)
            a = rng.uniform(0.5, 3.0, K)
            assert abs(float(_mp_dirichlet(lw, a)) - stats.dirichlet.logpdf(w, a)) <= 1e-12 * max(1.0, abs(float(_mp_dirichlet(lw, a))))
            h = 1e-6
            J = np.empty((K - 1, K - 1))
            for j in range(K - 1):
                e = np.zeros(K - 1)
                e[j] = h
                J[:, j] = (ir.simplex_backward(z + e)[:-1] - ir.simplex_backward(z - e)[:-1]) / (2 * h)
            assert abs(float(lj) - np.linalg.slogdet(J)[1]) <= 1e-7, (K, float(lj), np.linalg.slogdet(J)[1])
            mu, s, eta = np.sort(rng.normal(0.0, 3.0, K)), rng.uniform(0.5, 2.0, K), 0.3
            lam = np.sort(rng.uniform(0.5, 10.0, K))
            lwm = [mp.log(mpf(float(v))) for v in w]
            for y in (-4.0, 0.2, 3.5):
                want = logsumexp(np.log(w) + stats.norm.logpdf(y, eta + mu, s))
                got = float(_mp_mixture("normal_mixture", y, mpf(eta), lwm, [mpf(v) for v in mu], [mpf(v) for v in s]))
                assert abs(got - want) <= 1e-13 * max(1.0, abs(want))
            for y in (0.0, 2.0, 11.0):
                want = logsumexp(np.log(w) + stats.poisson.logpmf(y, lam * np.exp(eta)))
                got = float(_mp_mixture("poisson_mixture", y, mpf(eta), lwm, [mpf(v) for v in lam], None))
                assert abs(got - want) <= 1e-13 * max(1.0, abs(want))


@pytest.mark.parametrize("cid", list(CASES))
def test_oracle_matches_the_mp_reference_and_central_differences(cid):
    from oracle import ir_numpy_mixture

    m = CASES[cid]()
    f = ir_numpy_mixture.make_logp(m)
    for q in _points(cid, m):
        lp, g = f(q)
        lp_mp, S = _mp_logp(m, q)
        assert np.isfinite(lp) and np.all(np.isfinite(g))
        assert abs(lp - lp_mp) <= 1e-13 * S, (cid, lp, lp_mp)
        g_mp = _mp_grad(m, q)
        assert np.max(np.abs(g - g_mp)) <= 1e-11 * max(1.0, np.max(np.abs(g_mp))), (cid, g, g_mp)
        if cid != "normal_k3_log_w_near_minus_700":
            gf = fd_grad(f, q)
            assert np.max(np.abs(g - gf)) <= 1e-6 * max(1.0, np.max(np.abs(g))), (cid, g, gf)


def _overflowing_poisson():
    """A Poisson mixture whose second rate lam e^eta overflows at b0 = 10: that component's density is 0 (l = -inf) while
    the first one's is finite, so the mixture's density is the first component's alone."""
    return _model("poisson_mixture", 2, [0.4, 0.6], [2.0, 1e306], None, "scalar")


def test_a_component_whose_density_underflows_to_zero_adds_nothing():
    from oracle import ir_numpy_mixture

    m = _overflowing_poisson()
    q = np.array([10.0])
    lp, g = ir_numpy_mixture.make_logp(m)(q)
    L = m.likelihoods[0]
    want = np.sum(np.log(0.4) + stats.poisson.logpmf(L.y, 2.0 * np.exp(10.0))) + stats.norm.logpdf(10.0)
    assert np.isfinite(lp) and np.all(np.isfinite(g)) and abs(lp - want) <= 1e-12 * abs(want)
    gw = np.sum(L.y - 2.0 * np.exp(10.0)) - 10.0
    assert abs(g[0] - gw) <= 1e-12 * abs(gw)


def test_the_oracle_covers_models_that_mix_old_and_new_factors():
    """A mixture next to a survival likelihood: the sum of the two oracles' parts."""
    from oracle import ir_numpy_mixture, ir_numpy_survival

    a = ir.mixture_ir("normal", 3, "dirichlet", 0, n_obs=40)
    b = ir.survival_regression_ir("weibull", "right_censored", n_obs=30)
    both = ModelIR(vars=a.vars + b.vars, priors=a.priors + b.priors, likelihoods=a.likelihoods + b.likelihoods)
    q = np.concatenate([a.initial_point(), b.initial_point()]) + 0.1
    lp, g = ir_numpy_mixture.make_logp(both)(q)
    la, ga = ir_numpy_mixture.make_logp(a)(q[:a.n])
    lb, gb = ir_numpy_survival.make_logp(b)(q[a.n:])
    assert abs(lp - (la + lb)) <= 1e-12 * abs(lp)
    np.testing.assert_allclose(g, np.concatenate([ga, gb]), rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------------
# the support rule, through validate() and the C ABI
# ------------------------------------------------------------------------------------------------------------------------
def _edit(m, fn):
    m = copy.deepcopy(m)
    fn(m)
    return m


def _lik(**kw):
    return lambda m: m.likelihoods.__setitem__(0, dataclasses.replace(m.likelihoods[0], **kw))


VALIDATE_CASES = [
    ("k1", lambda: _model("normal_mixture", 1, [1.0], [0.0], 1.0), ir.MIX_K),
    ("y_nan", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.likelihoods[0].y.__setitem__(3, np.nan)), ir.MIX_Y_NORMAL),
    ("y_half", lambda: _edit(ir.mixture_ir("poisson", 2), lambda m: m.likelihoods[0].y.__setitem__(3, 1.5)), ir.ZI_Y),
    ("w_sum", lambda: _model("normal_mixture", 3, [0.3, 0.3, 0.3], "ordered", 1.0), ir.MIX_WEIGHTS),
    ("w_negative", lambda: _model("normal_mixture", 2, [1.2, -0.2], "ordered", 1.0), ir.MIX_WEIGHTS),
    ("w_length", lambda: _model("normal_mixture", 3, [0.5, 0.5], "ordered", 1.0), ir.MIX_WEIGHTS),
    ("w_not_simplex", lambda: _edit(ir.mixture_ir("normal", 3), _lik(weights=Ref("mu_ordered__"))), ir.MIX_WEIGHTS),
    ("mu_log", lambda: _model("normal_mixture", 3, "var", "log", 1.0), ir.MIX_MU),
    ("mu_inf", lambda: _model("normal_mixture", 2, "var", [0.0, np.inf], 1.0), ir.MIX_MU),
    ("lam_real", lambda: _model("poisson_mixture", 3, "var", "ordered"), ir.MIX_LAM),
    ("lam_zero", lambda: _model("poisson_mixture", 2, "var", [0.0, 1.0]), ir.MIX_LAM),
    ("sigma_missing", lambda: _model("normal_mixture", 2, "var", "ordered", None), ir.MIX_SIGMA),
    ("sigma_zero", lambda: _model("normal_mixture", 2, "var", "ordered", [1.0, 0.0]), ir.MIX_SIGMA),
    ("sigma_real_var", lambda: _edit(ir.mixture_ir("normal", 3), _lik(sigma=Ref("mu_ordered__"))), ir.MIX_SIGMA),
    ("sigma_per_obs", lambda: _edit(ir.mixture_ir("normal", 3), _lik(sigma=np.ones(300))), ir.MIX_SIGMA),
    ("slot_alpha", lambda: _edit(ir.mixture_ir("poisson", 2), _lik(alpha=2.0)), ir.MIX_SLOTS),
    ("slot_sigma", lambda: _edit(ir.mixture_ir("poisson", 2), _lik(sigma=1.0)), ir.MIX_SLOTS),
    ("slot_psi", lambda: _edit(ir.mixture_ir("normal", 2), _lik(psi=0.5)), ir.MIX_SLOTS),
    ("slot_lower", lambda: _edit(ir.mixture_ir("normal", 2), _lik(lower=-10.0)), ir.MIX_SLOTS),
    ("slot_cutpoints", lambda: _edit(ir.mixture_ir("normal", 2), _lik(cutpoints=np.zeros(1))), ir.MIX_SLOTS),
    ("simplex_as_term", lambda: _edit(ir.mixture_ir("normal", 2), _lik(terms=[Term([("w_simplex__", None)])])),
     ir.SIMPLEX_USE),
    ("simplex_as_prior_param", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.priors.__setitem__(
        1, Prior("normal", "mu_ordered__", (0.0, Ref("w_simplex__"))))), ir.SIMPLEX_USE),
    ("simplex_as_components", lambda: _edit(ir.mixture_ir("normal", 2), _lik(components=Ref("w_simplex__"))),
     ir.SIMPLEX_USE),
    ("simplex_as_sigma", lambda: _edit(ir.mixture_ir("normal", 2), _lik(sigma=Ref("w_simplex__"))), ir.SIMPLEX_USE),
    ("simplex_as_ar1", lambda: _edit(ir.mixture_ir("normal", 3), lambda m: m.ar1.append(ir.AR1("w_simplex__"))),
     ir.SIMPLEX_USE),
    ("simplex_in_deterministic", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.deterministics.append(
        ir.Deterministic("d", 1, [Term([("w_simplex__", None)])]))), ir.SIMPLEX_USE),
    ("simplex_in_linear", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.priors.__setitem__(
        1, Prior("normal", "mu_ordered__", (ir.Linear([Term([("w_simplex__", None)])]), 10.0)))), ir.SIMPLEX_USE),
    ("simplex_as_cutpoints", lambda: _edit(ir.mixture_ir("normal", 3), lambda m: m.likelihoods.append(
        Likelihood("ordered_logistic", np.array([0.0, 1.0, 2.0]), [], cutpoints=Ref("w_simplex__")))), ir.SIMPLEX_USE),
    ("simplex_as_psi", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.likelihoods.append(
        Likelihood("zero_inflated_poisson", np.array([0.0, 1.0]), [], psi=Ref("w_simplex__")))), ir.SIMPLEX_USE),
    ("simplex_normal_prior", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.priors.__setitem__(
        0, Prior("normal", "w_simplex__", (0.0, 1.0)))), ir.SIMPLEX_PRIOR),
    ("simplex_two_priors", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.priors.append(
        Prior("dirichlet", "w_simplex__", (1.0,)))), ir.SIMPLEX_PRIOR),
    ("simplex_no_prior", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.priors.pop(0)), ir.SIMPLEX_PRIOR),
    ("dirichlet_off_simplex", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.priors.__setitem__(
        1, Prior("dirichlet", "mu_ordered__", (1.0,)))), ir.DIRICHLET_VAR),
    ("dirichlet_a_zero", lambda: _edit(ir.mixture_ir("normal", 2), lambda m: m.priors.__setitem__(
        0, Prior("dirichlet", "w_simplex__", (0.0,)))), ir.DIRICHLET_A),
    ("dirichlet_a_length", lambda: _edit(ir.mixture_ir("normal", 3), lambda m: m.priors.__setitem__(
        0, Prior("dirichlet", "w_simplex__", (np.ones(2),)))), ir.DIRICHLET_A),
    ("dirichlet_a_unequal", lambda: _edit(ir.mixture_ir("normal", 3), lambda m: m.priors.__setitem__(
        0, Prior("dirichlet", "w_simplex__", (np.array([1.0, 2.0, 1.0]),)))), ir.DIRICHLET_A),
    ("weights_on_normal", lambda: _edit(ir.mixture_ir("normal", 2), _lik(dist="normal", sigma=1.0)),
     "weights and components belong to the mixture likelihoods"),
]


@pytest.mark.parametrize("case", VALIDATE_CASES, ids=[c[0] for c in VALIDATE_CASES])
def test_validate_refuses_each_clause_of_the_support_rule(case):
    _, build, msg = case
    with pytest.raises(ValueError, match=None) as e:
        build().validate()
    assert msg in str(e.value), (msg, str(e.value))


def test_existing_refusals_keep_their_words():
    m = _edit(ir.mixture_ir("normal", 2), lambda m: m.likelihoods.append(Likelihood("normal", np.zeros(3), [], sigma=Ref("mu_ordered__"))))
    with pytest.raises(ValueError, match="likelihood sigma must be a scalar variable"):
        m.validate()


def test_model_create_refuses_malformed_mixture_tables_through_the_c_abi():
    """prepare_ir makes the checks of validate(), with the same words, for callers of the C ABI."""
    nd = lambda: ir.mixture_ir("normal", 3, "dirichlet", 1, n_obs=40)  # noqa: E731  vars: w(2), mu(3), sigma(3), beta(1)
    pc = lambda: ir.mixture_ir("poisson", 3, "const", 0, n_obs=40)  # noqa: E731

    def mix(b, **kw):
        return lambda low: low.liks[0]["mix"][b].update(**kw)

    def y_at(v):
        def edit(low):
            low.liks[0]["y"] = low.liks[0]["y"].copy()
            low.liks[0]["y"][2] = v
        return edit

    def prior(k, **kw):
        def edit(low):
            dist, var, pars = low.priors[k]
            low.priors[k] = (kw.get("dist", dist), kw.get("var", var), kw.get("pars", pars))
        return edit

    cases = [
        (nd, lambda low: low.liks[0].update(nu=1.0), ir.MIX_K),
        (nd, y_at(np.inf), ir.MIX_Y_NORMAL), (pc, y_at(0.5), ir.ZI_Y),
        (nd, lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_CONST, sigma_value=1.0), ir.MIX_SLOTS),
        (pc, mix(0, coef=np.array([0.3, 0.3, 0.3])), ir.MIX_WEIGHTS),
        (pc, mix(0, coef=np.array([1.1, 0.2, -0.3])), ir.MIX_WEIGHTS),
        (nd, mix(0, factors=[(2, 3, None)]), ir.MIX_WEIGHTS),
        (nd, mix(1, factors=[(5, 3, None)]), ir.MIX_MU),
        (pc, mix(1, coef=np.array([1.0, 0.0, 2.0])), ir.MIX_LAM),
        (nd, mix(2, coef=np.array([1.0, 0.0, 2.0]), factors=[]), ir.MIX_SIGMA),
        (nd, mix(2, factors=[(2, 3, None)]), ir.MIX_SIGMA),
        (nd, mix(1, factors=[(0, 2, None)]), ir.SIMPLEX_USE),
        (nd, lambda low: low.liks[0]["terms"].append(dict(coef=None, factors=[(0, 2, None)])), ir.SIMPLEX_USE),
        (nd, prior(1, pars=[(0, 0.0, -1), (1, 0.0, 0), (0, 0.0, -1)]), ir.SIMPLEX_USE),
        (nd, lambda low: low.ar1.append((0, (0, 1.0, -1), (0, 1.0, -1), 1.0)), ir.SIMPLEX_USE),
        (nd, prior(0, dist=ir.PRIOR_DISTS["normal"][0], pars=[(0, 0.0, -1), (0, 1.0, -1), (0, 0.0, -1)]), ir.SIMPLEX_PRIOR),
        (nd, lambda low: low.priors.pop(0), ir.SIMPLEX_PRIOR),
        (nd, lambda low: low.priors.append(low.priors[0]), ir.SIMPLEX_PRIOR),
        (nd, prior(1, dist=ir.PRIOR_DISTS["dirichlet"][0], pars=[(0, 1.0, -1)] * 3), ir.DIRICHLET_VAR),
        (nd, prior(0, pars=[(0, -1.0, -1)] + [(0, 0.0, -1)] * 2), ir.DIRICHLET_A),
    ]
    for builder, edit, msg in cases:
        err = refusal_after_edit(builder, edit)
        assert err is not None and msg in err, (msg, err)


def test_the_eta_free_mixture_is_accepted_but_an_empty_predictor_stays_refused_elsewhere():
    low = ir.lower(ir.mixture_ir("poisson", 2, "const", 0))
    assert low.liks[0]["terms"] == [] and create_raw(low) is None
    low = ir.lower(ir.mixture_ir("normal", 2, "dirichlet", 1))
    low.liks[0].update(dist=ir.LIK_DISTS["normal"], terms=[], sigma_kind=ir.SIGMA_CONST, sigma_value=1.0)
    assert "no linear-predictor terms" in create_raw(low)


# ------------------------------------------------------------------------------------------------------------------------
# tables, constrain, routing, the sampler's data groups
# ------------------------------------------------------------------------------------------------------------------------
def test_lowered_tables_hold_the_transform_the_prior_and_the_blocks():
    m = ir.mixture_ir("normal", 4, "dirichlet", 2)
    low = ir.lower(m)
    off = m.offsets()
    assert tuple(low.vars[0]) == (0, 3, 5)
    assert low.priors[0] == (11, 0, [(0, 1.0, -1), (0, 0.0, -1), (0, 0.0, -1)])
    L = low.liks[0]
    assert L["dist"] == 24 and L["nu"] == 4.0 and L["sigma_kind"] == ir.SIGMA_NONE and len(L["terms"]) == 1
    assert [b["factors"] for b in L["mix"]] == [[(0, 3, None)], [(off["mu_ordered__"], 4, None)], [(off["sigma_log__"], 4, None)]]
    c = ir.lower(_model("normal_mixture", 3, [0.2, 0.3, 0.5], [0.0, 1.0, 2.0], 1.5))
    assert [b["factors"] for b in c.liks[0]["mix"]] == [[], [], []]
    np.testing.assert_array_equal(c.liks[0]["mix"][2]["coef"], [1.5, 1.5, 1.5])
    p = ir.lower(ir.mixture_ir("poisson", 3, "const"))
    assert p.liks[0]["dist"] == 25 and len(p.liks[0]["mix"]) == 2
    np.testing.assert_allclose(p.liks[0]["mix"][0]["coef"].sum(), 1.0)


def test_constrain_returns_the_k_weights():
    from pymc_b200 import engine

    m = ir.mixture_ir("normal", 2, "dirichlet")
    q = m.initial_point() + np.random.default_rng(0).normal(0.0, 2.0, (4, 5, m.n))
    for out in (m.constrain(q), engine._ir_spec(m).constrain(q)):
        w = out["w"]
        assert w.shape == (4, 5, 2)
        np.testing.assert_allclose(w.sum(-1), 1.0, rtol=1e-15)
        np.testing.assert_allclose(w, ir.simplex_backward(q[..., :1]), rtol=1e-15)


def test_specialise_declines_and_fuse_design_columns_keeps_the_blocks():
    from oracle import ir_numpy_mixture

    m = ir.mixture_ir("poisson", 3, "dirichlet", 2)
    assert ir.specialise(m) is None and ir.specialise(m, extended=True) is None
    L = m.likelihoods[0]
    X = L.terms[0].coef
    cols = dataclasses.replace(m, likelihoods=[dataclasses.replace(L, terms=[
        Term([("beta", np.full(len(L.y), k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(2)])])
    fused = ir.fuse_design_columns(cols)
    F = fused.likelihoods[0]
    assert ir.is_design(F.terms[0]) and F.weights == L.weights and F.components == L.components
    q = m.initial_point() + 0.2
    (a, ga), (b, gb) = ir_numpy_mixture.make_logp(m)(q), ir_numpy_mixture.make_logp(fused)(q)
    assert abs(a - b) <= 1e-12 * abs(b) and np.allclose(ga, gb, rtol=1e-11, atol=1e-11)


def _scipy_pointwise(m, P, X=None):
    L = m.likelihoods[0]
    w = P["w"] if "w" in P else np.asarray(L.weights)
    eta = X @ np.atleast_1d(P["beta"]) if X is not None else 0.0
    with np.errstate(divide="ignore"):
        if L.dist == "normal_mixture":
            comp = stats.norm.logpdf(L.y[:, None], (eta + 0.0 * L.y)[:, None] + P["mu"], P["sigma"])
        else:
            comp = stats.poisson.logpmf(L.y[:, None], np.exp(eta + 0.0 * L.y)[:, None] * P["lam"])
        return logsumexp(np.log(w) + comp, axis=1)


def test_sampler_records_the_mixture_log_likelihood():
    """The sampler on the oracle-backed stand-in: the posterior holds the K weights and the log_likelihood group the
    mixture density of every observation."""
    from b200_helpers import OracleEngine
    from oracle import ir_numpy_mixture
    from pymc_b200 import engine, sampling

    m = ir.mixture_ir("normal", 3, "dirichlet", 2, n_obs=50)

    class IrStandIn(OracleEngine):
        def __init__(self, model):
            self.ir, self.spec = model, engine._ir_spec(model)
            self.n, self.f = model.n, ir_numpy_mixture.make_logp(model)

        def pointwise_loglik(self, draws, lik=0):
            q = np.asarray(draws)
            L = self.ir.likelihoods[lik]
            out = np.empty(q.shape[:-1] + (len(L.y),))
            for ix in np.ndindex(*q.shape[:-1]):
                out[ix] = self.f.loglik(L, self.f.constrained(q[ix])[0], q[ix])
            return out

    res = sampling.sample_b200_nuts(5, tune=10, chains=2, random_seed=4, model=IrStandIn(m), momentum="numpy",
                                    keep_untransformed=True, idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
    assert res.posterior["w"].shape == (2, 5, 3)
    np.testing.assert_allclose(res.posterior["w"].sum(-1), 1.0, rtol=1e-14)
    ll = res.log_likelihood["y"]
    assert ll.shape == (2, 5, 50)
    X = m.likelihoods[0].terms[0].coef
    for c in range(2):
        for d in range(5):
            P = {k: res.posterior[k][c, d] for k in ("w", "mu", "sigma", "beta")}
            np.testing.assert_allclose(ll[c, d], _scipy_pointwise(m, P, X), rtol=1e-11, atol=1e-11)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
BUILDERS = {
    "normal_dirichlet": lambda: ir.mixture_ir("normal", 3, "dirichlet"),                           # n = 8: warp
    "normal_const_design": lambda: ir.mixture_ir("normal", 2, "const", 3),
    "poisson_dirichlet_design": lambda: ir.mixture_ir("poisson", 3, "dirichlet", 2),
    "poisson_const": lambda: ir.mixture_ir("poisson", 5, "const"),
    "normal_dirichlet_cta": lambda: ir.mixture_ir("normal", 3, "dirichlet", 260, n_obs=600),       # n = 268: CTA
    "normal_k130_cta": lambda: ir.mixture_ir("normal", 130, "dirichlet", 0, n_obs=600),            # n = 389: CTA
}


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(CASES))
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid):
    """Chain = warp, then chain = CTA forced: each against the mp reference and the oracle, bit-identical when repeated."""
    from oracle import ir_numpy_mixture
    from pymc_b200 import engine

    m = CASES[cid]()
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = ir_numpy_mixture.make_logp(m)
    Q = _points(cid, m)
    ref = [_mp_logp(m, q) for q in Q]
    g_mp = np.array([_mp_grad(m, q) for q in Q])
    go = np.array([f(q)[1] for q in Q])
    for team, (lp, g) in logp_at_both_team_shapes(cm, Q).items():
        assert np.all(np.isfinite(lp)) and np.all(np.isfinite(g)), (cid, team)
        for k, (lp_mp, S) in enumerate(ref):
            assert abs(lp[k] - lp_mp) <= 1e-13 * S, (cid, team, lp[k], lp_mp)
            for gr in (g_mp[k], go[k]):
                assert np.max(np.abs(g[k] - gr)) <= 1e-12 * max(1.0, np.max(np.abs(gr))), (cid, team, g[k], gr)


@pytest.mark.gpu
def test_device_skips_a_component_whose_density_underflows_to_zero():
    from oracle import ir_numpy_mixture
    from pymc_b200 import engine

    m = _overflowing_poisson()
    cm = engine.CompiledModel(m, specialise=False)
    Q = np.array([[10.0], [9.5], [0.3]])
    f = ir_numpy_mixture.make_logp(m)
    for team, (lp, g) in logp_at_both_team_shapes(cm, Q).items():
        for k, q in enumerate(Q):
            lo, go = f(q)
            assert np.isfinite(lp[k]) and np.all(np.isfinite(g[k])), (team, q)
            assert abs(lp[k] - lo) <= 1e-12 * abs(lo) and np.max(np.abs(g[k] - go)) <= 1e-12 * max(1.0, np.max(np.abs(go)))
    ll = cm.pointwise_loglik(Q)
    assert np.all(np.isfinite(ll))
    np.testing.assert_allclose(ll[0], np.log(0.4) + stats.poisson.logpmf(m.likelihoods[0].y, 2.0 * np.exp(10.0)), rtol=1e-11)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_device_function_matches_the_oracle_on_the_builders(name):
    from oracle import ir_numpy_mixture
    from pymc_b200 import engine

    m = BUILDERS[name]()
    cm = engine.CompiledModel(m)  # default path: no hand kernel takes it
    assert cm.spec.name == "ir" and (m.n > 256) == name.endswith("cta")
    f = ir_numpy_mixture.make_logp(m)
    Q = m.initial_point() + np.random.default_rng(0).uniform(-1.0, 1.0, (9, m.n))
    lp, g = cm.logp_dlogp(Q)
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12
    assert np.max(np.abs(g - go) / np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))) <= 1e-11
    lp2, g2 = cm.logp_dlogp(Q)
    assert np.array_equal(lp, lp2) and np.array_equal(g, g2)


@pytest.mark.gpu
@pytest.mark.parametrize("name,eps", [("normal_dirichlet", 0.05), ("poisson_dirichlet_design", 0.05),
                                      ("normal_dirichlet_cta", 0.005)])
def test_fixed_step_nuts_matches_the_oracle_sampler(name, eps):
    from oracle import ir_numpy_mixture

    m = BUILDERS[name]()
    fixed_step_against_oracle(m, ir_numpy_mixture.make_logp(m), eps)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle():
    from oracle import ir_numpy_mixture

    m = ir.mixture_ir("normal", 3, "dirichlet", 1)
    fixed_step_against_oracle(m, ir_numpy_mixture.make_logp(m), 0.05, dense_cov=random_dense_cov(m.n, 2, 0.05, 0.05, 12),
                              C=2, T=10)


@pytest.mark.gpu
def test_adaptive_normal_mixture_run_matches_the_oracle_posterior():
    """64 device chains against 8 oracle chains on the 3-component Normal mixture with Dirichlet weights: posterior means
    within 5 SE, standard deviations within 25 %, divergences below 2 %."""
    from oracle import ir_numpy_mixture

    m = ir.mixture_ir("normal", 3, "dirichlet")
    adaptive_against_oracle(m, ir_numpy_mixture.make_logp(m), chain_seed=29, spread=0.3, philox_seed=7, oracle_seed=300,
                            se_bound=5.0, max_divergence=0.02)


@pytest.mark.gpu
def test_pointwise_log_likelihood_and_the_log_likelihood_group_match_scipy():
    import pymc_b200
    from pymc_b200 import engine

    for m in (ir.mixture_ir("normal", 3, "dirichlet", 2, n_obs=120), ir.mixture_ir("poisson", 4, "const", 1, n_obs=120),
              _model("normal_mixture", 3, [0.5, 0.0, 0.5], [-2.0, 0.0, 2.0], 1.3, "design", N=30)):
        cm = engine.CompiledModel(m, specialise=False)
        q = m.initial_point() + np.random.default_rng(4).uniform(-0.5, 0.5, (2, 3, m.n))
        ll = cm.pointwise_loglik(q)
        L = m.likelihoods[0]
        assert ll.shape == (2, 3, len(L.y)) and np.all(np.isfinite(ll))
        post = m.constrain(q)
        X = L.terms[0].coef if L.terms else None
        for ix in np.ndindex(2, 3):
            P = {k: v[ix] for k, v in post.items()}
            P.setdefault("mu", L.components)
            P.setdefault("lam", L.components)
            P.setdefault("sigma", L.sigma)
            np.testing.assert_allclose(ll[ix], _scipy_pointwise(m, P, X), rtol=1e-11, atol=1e-11)
    m = ir.mixture_ir("normal", 3, "dirichlet", 2, n_obs=80)
    res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, keep_untransformed=True,
                                     idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
    ll = res.log_likelihood["y"]
    assert ll.shape == (4, 20, 80) and res.posterior["w"].shape == (4, 20, 3)
    X = m.likelihoods[0].terms[0].coef
    for c in range(4):
        for d in range(0, 20, 5):
            P = {k: res.posterior[k][c, d] for k in ("w", "mu", "sigma", "beta")}
            np.testing.assert_allclose(ll[c, d], _scipy_pointwise(m, P, X), rtol=1e-11, atol=1e-11)
