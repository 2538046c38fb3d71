"""Gaussian processes in the model IR: spectral (HSGP) terms and the InverseGamma prior.

- ``hsgp_basis`` with the spectral densities reproduces the exact ExpQuad / Matern 5/2 / Matern 3/2 kernels of PyMC's
  cov.py as Phi diag(S) Phi^T, in 1-D and 2-D ARD (every constant of S is pinned: a wrong factor gives O(1) errors).
- oracle/ir_numpy_hsgp.py against a 40-digit mpmath evaluation and central differences, at points where s_k underflows,
  at extreme lengthscales, in 1-D and 2-D, with constant and random ls and amplitude.
- ``validate()`` refuses every malformed spectral term, and ``prepare_ir`` in the same words through the C ABI.
- constant ls and amplitude lower to a plain design term; Deterministics, constant_data, specialise and
  fuse_design_columns.
- on the GPU: the device logp and gradient against the mp reference and the oracle at both team shapes, bit-identical
  when repeated; the pointwise log-likelihood against scipy; fixed-step and adaptive NUTS against the oracle sampler.
"""
from __future__ import annotations

import copy

import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import stats
from b200_helpers import (adaptive_against_oracle, fd_grad, fixed_step_against_oracle, logp_at_both_team_shapes,
                          random_dense_cov, refusal_after_edit)

from pymc_b200 import ir
from pymc_b200.ir import Likelihood, ModelIR, Prior, Ref, Spectral, Term, Var

MP_DPS = 40


# ---- basis and spectral densities against the exact kernels ------------------------------------------------------------
def exact_kernel(cov, X, ls):
    r2 = np.sum(((X[:, None, :] - X[None, :, :]) / np.asarray(ls)) ** 2, axis=-1)
    if cov == "expquad":
        return np.exp(-0.5 * r2)
    r = np.sqrt(r2)
    if cov == "matern52":
        return (1.0 + np.sqrt(5.0) * r + 5.0 / 3.0 * r2) * np.exp(-np.sqrt(5.0) * r)
    return (1.0 + np.sqrt(3.0) * r) * np.exp(-np.sqrt(3.0) * r)


def kernel_error(cov, X, ls, m, c):
    Phi, omega, _, _ = ir.hsgp_basis(X, m, c=c)
    D = omega.shape[1]
    s = np.exp(ir.spectral_log_scale(cov, omega, np.broadcast_to(np.asarray(ls, dtype=np.float64), (D,)), 1.0))
    return np.max(np.abs((Phi * s**2) @ Phi.T - exact_kernel(cov, X.reshape(len(X), -1), ls)))


@pytest.mark.parametrize("cov,c,m,tol", [("expquad", 3.0, 100, 4e-15), ("matern52", 5.0, 2000, 1.2e-10),
                                         ("matern32", 5.0, 2000, 5e-7)])
def test_basis_reproduces_the_exact_kernel_in_one_dimension(cov, c, m, tol):
    X = np.linspace(-1.0, 1.0, 101)[:, None]
    assert kernel_error(cov, X, 0.3, m, c) <= tol


@pytest.mark.parametrize("cov,c,m,tol", [("expquad", 3.0, 60, 1.5e-6), ("matern52", 4.0, 150, 7e-6),
                                         ("matern32", 4.0, 150, 2.5e-4)])
def test_basis_reproduces_the_exact_ard_kernel_in_two_dimensions(cov, c, m, tol):
    X = np.random.default_rng(3).uniform(-1.0, 1.0, (60, 2))
    assert kernel_error(cov, X, [0.4, 0.7], [m, m], c) <= tol


def test_a_wrong_constant_is_an_order_one_error():
    X = np.linspace(-1.0, 1.0, 101)[:, None]
    Phi, omega, _, _ = ir.hsgp_basis(X, 2000, c=5.0)
    s2 = np.exp(2.0 * ir.spectral_log_scale("matern52", omega, np.array([0.3]), 1.0))
    assert np.max(np.abs((Phi * s2 * 1.1) @ Phi.T - exact_kernel("matern52", X, 0.3))) > 0.05


def test_basis_layout_follows_meshgrid_and_drop_first():
    X = np.random.default_rng(1).uniform(2.0, 6.0, (20, 2))
    Phi, omega, centre, L = ir.hsgp_basis(X, [3, 4], c=1.5)
    assert Phi.shape == (20, 12) and omega.shape == (12, 2)
    np.testing.assert_allclose(centre, 0.5 * (X.max(0) + X.min(0)))
    np.testing.assert_allclose(L, 1.5 * 0.5 * (X.max(0) - X.min(0)))
    J = omega * 2.0 * L / np.pi
    np.testing.assert_allclose(J[:4], [[1, 1], [2, 1], [3, 1], [1, 2]])  # the first dimension varies fastest
    Phi2, omega2, _, L2 = ir.hsgp_basis(X, [3, 4], L=L, drop_first=True)
    np.testing.assert_array_equal(Phi2, Phi[:, 1:])
    np.testing.assert_array_equal(omega2, omega[1:])


# ---- the oracle against a high-precision reference -------------------------------------------------------------------
def small_model(cov, D, ls_kind, amp_kind, N=7, m=5, c=1.3, seed=2):
    """y ~ Normal(b0 + Phi (z * s), sigma) with b0 ~ Normal(0, 1), z ~ Normal(0, 1)^M, sigma ~ HalfNormal(1); ls: 'var'
    (ARD, InverseGamma(3, 2)), 'iso' (one variable), or constants; amp: 'var' (HalfNormal(1.5)) or a constant."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-2.0, 2.0, (N, D))
    Phi, omega, _, _ = ir.hsgp_basis(X, [m] * D, c=c)
    M = Phi.shape[1]
    vars_ = [Var("b0", "b0", 1), Var("z", "z", M), Var("sigma_log__", "sigma", 1, "log")]
    priors = [Prior("normal", "b0", (0.0, 1.0)), Prior("normal", "z", (0.0, 1.0)), Prior("halfnormal", "sigma_log__", (1.0,))]
    ls, amp = (np.linspace(0.6, 0.9, D) if D > 1 else 0.7), 1.3
    if ls_kind in ("var", "iso"):
        vars_.append(Var("ell_log__", "ell", D if ls_kind == "var" else 1, "log"))
        priors.append(Prior("inversegamma", "ell_log__", (3.0, 2.0)))
        ls = Ref("ell_log__")
    if amp_kind == "var":
        vars_.append(Var("eta_log__", "eta", 1, "log"))
        priors.append(Prior("halfnormal", "eta_log__", (1.5,)))
        amp = Ref("eta_log__")
    y = rng.normal(0.0, 1.0, N)
    t = Term([("z", None)], coef=Phi, spectral=Spectral(cov, omega, ls, amp))
    return ModelIR(name=f"small_{cov}_{D}_{ls_kind}_{amp_kind}", vars=vars_, priors=priors,
                   likelihoods=[Likelihood("normal", y, [Term([("b0", None)]), t], sigma=Ref("sigma_log__"))])


CASES = {
    "expquad_1d_var": ("expquad", 1, "var", "var"),
    "expquad_2d_ard": ("expquad", 2, "var", "var"),
    "expquad_2d_iso": ("expquad", 2, "iso", "const"),
    "matern52_1d_var": ("matern52", 1, "var", "var"),
    "matern52_2d_ard": ("matern52", 2, "var", "const"),
    "matern32_1d_const_ls": ("matern32", 1, "const", "var"),
    "matern32_2d_ard": ("matern32", 2, "var", "var"),
}


def case_points(m):
    """The initial point moved at random, then the lengthscale near both extremes: small, and large enough that
    ExpQuad's s_k underflows for all but the first few k."""
    rng = np.random.default_rng(11)
    Q = [m.initial_point() + rng.uniform(-0.8, 0.8, m.n) for _ in range(2)]
    if any(v.name == "ell_log__" for v in m.vars):
        o = m.offsets()["ell_log__"]
        for lv in (np.log(1e-3), np.log(60.0), np.log(400.0)):
            q = Q[0].copy()
            q[o : o + m.var("ell_log__").size] = lv
            Q.append(q)
    return np.array(Q)


def _mp_logp(m, q):
    """The log-density of a small_model at q (unconstrained) in mpmath, every constant included."""
    mp.dps = MP_DPS
    off = m.offsets()
    x = {}
    lp = mpf(0)
    for v in m.vars:
        z = [a if isinstance(a, mpf) else mpf(float(a)) for a in q[off[v.name] : off[v.name] + v.size]]
        if v.transform == "log":
            lp += sum(z)
            z = [mp.exp(a) for a in z]
        x[v.name] = z
    for p in m.priors:
        for xv in x[p.var]:
            if p.dist == "normal":
                mu, sg = (mpf(float(a)) for a in p.params)
                lp += -((xv - mu) / sg) ** 2 / 2 - mp.log(sg) - mp.log(2 * mp.pi) / 2
            elif p.dist == "halfnormal":
                sg = mpf(float(p.params[0]))
                lp += -(xv / sg) ** 2 / 2 - mp.log(sg) + mp.log(2 / mp.pi) / 2
            else:  # inversegamma
                a, b = (mpf(float(c)) for c in p.params)
                lp += a * mp.log(b) - mp.loggamma(a) - (a + 1) * mp.log(xv) - b / xv
    L = m.likelihoods[0]
    t = L.terms[1]
    sp = t.spectral
    om = np.asarray(sp.omega)
    M, D = om.shape
    ls = x["ell_log__"] if isinstance(sp.ls, Ref) else [mpf(float(a)) for a in np.broadcast_to(np.ravel(sp.ls), (D,))]
    ls = ls * D if len(ls) == 1 else ls
    amp = x["eta_log__"][0] if isinstance(sp.amplitude, Ref) else mpf(float(sp.amplitude))
    s = []
    for k in range(M):
        Q = sum((ls[d] * mpf(float(om[k, d]))) ** 2 for d in range(D))
        pl = mp.fprod(ls)
        if sp.cov == "expquad":
            S = (2 * mp.pi) ** (mpf(D) / 2) * pl * mp.exp(-Q / 2)
        elif sp.cov == "matern52":
            S = (2 ** D * mp.pi ** (mpf(D) / 2) * mp.gamma(mpf(D + 5) / 2) * mpf(5) ** mpf(2.5) / (mpf(3) / 4 * mp.sqrt(mp.pi))
                 * pl * (5 + Q) ** (-mpf(D + 5) / 2))
        else:
            S = (2 ** D * mp.pi ** (mpf(D) / 2) * mp.gamma(mpf(D + 3) / 2) * mpf(3) ** mpf(1.5) / (mpf(1) / 2 * mp.sqrt(mp.pi))
                 * pl * (3 + Q) ** (-mpf(D + 3) / 2))
        s.append(amp * mp.sqrt(S))
    Phi = np.asarray(t.coef)
    sg = x["sigma_log__"][0]
    for i in range(len(L.y)):
        f = x["b0"][0] + mp.fsum(mpf(float(Phi[i, k])) * s[k] * x["z"][k] for k in range(M))
        lp += -((mpf(float(L.y[i])) - f) / sg) ** 2 / 2 - mp.log(sg) - mp.log(2 * mp.pi) / 2
    return lp


def mp_reference(m, Q):
    """(logp, gradient) at each point: mp values, and mp central differences with h = 1e-15 at 40 digits."""
    lps, gs = [], []
    h = mpf("1e-15")
    for q in Q:
        lps.append(float(_mp_logp(m, q)))
        g = np.empty(m.n)
        for j in range(m.n):
            qp, qm = [mpf(float(a)) for a in q], [mpf(float(a)) for a in q]
            qp[j] += h
            qm[j] -= h
            g[j] = float((_mp_logp(m, qp) - _mp_logp(m, qm)) / (2 * h))
        gs.append(g)
    return np.array(lps), np.array(gs)


def assert_close(lp, g, lp_ref, g_ref, tol, what):
    assert np.all(np.abs(lp - lp_ref) <= tol * np.maximum(1.0, np.abs(lp_ref))), what
    scale = np.maximum(1.0, np.max(np.abs(g_ref), axis=1, keepdims=True))
    assert np.all(np.abs(g - g_ref) <= tol * scale), (what, np.max(np.abs(g - g_ref) / scale))


@pytest.mark.parametrize("cid", list(CASES))
def test_oracle_matches_the_mp_reference_and_central_differences(cid):
    from oracle import ir_numpy_hsgp

    m = small_model(*CASES[cid])
    f = ir_numpy_hsgp.make_logp(m)
    Q = case_points(m)
    lp_mp, g_mp = mp_reference(m, Q)
    lo = np.array([f(q)[0] for q in Q])
    go = np.array([f(q)[1] for q in Q])
    assert np.all(np.isfinite(lo)) and np.all(np.isfinite(go))
    assert_close(lo, go, lp_mp, g_mp, 1e-12, cid)
    for q, g in zip(Q[:2], go[:2]):
        np.testing.assert_allclose(g, fd_grad(f, q), rtol=1e-6, atol=1e-6 * max(1.0, np.max(np.abs(g))))


def test_underflowing_scales_add_nothing_and_make_no_nan():
    from oracle import ir_numpy_hsgp

    m = small_model("expquad", 1, "var", "var", m=12)
    q = case_points(m)[-1]
    x = m.constrain(q)
    s = ir.spectral_weights(m, m.likelihoods[0].terms[1], x)
    assert np.sum(s == 0.0) >= 6 and np.all(np.isfinite(s))
    lp, g = ir_numpy_hsgp.make_logp(m)(q)
    assert np.isfinite(lp) and np.all(np.isfinite(g))


# ---- refusals ----------------------------------------------------------------------------------------------------------
def _spectral(m):
    return m.likelihoods[0].terms[1]


def _edit(fn):
    def build():
        m = small_model("expquad", 2, "var", "var")
        fn(m)
        return m
    return build


REFUSALS = [
    ("phi_shape", lambda m: setattr(_spectral(m), "coef", _spectral(m).coef[:, 1:]), ir.SPEC_PHI),
    ("phi_rows", lambda m: setattr(_spectral(m), "coef", _spectral(m).coef[1:]), ir.SPEC_PHI),
    ("phi_nan", lambda m: _spectral(m).coef.__setitem__((0, 0), np.nan), ir.SPEC_PHI),
    ("z_indexed", lambda m: setattr(_spectral(m), "factors", [("z", np.zeros(7, dtype=np.int32))]), ir.SPEC_Z),
    ("z_transformed", lambda m: setattr(m.var("z"), "transform", "log"), ir.SPEC_Z),
    ("cov", lambda m: setattr(_spectral(m).spectral, "cov", "ratquad"), ir.SPEC_COV),
    ("omega_shape", lambda m: setattr(_spectral(m).spectral, "omega", _spectral(m).spectral.omega[1:]), ir.SPEC_OMEGA),
    ("omega_negative", lambda m: _spectral(m).spectral.omega.__setitem__((1, 0), -0.5), ir.SPEC_OMEGA),
    ("omega_inf", lambda m: _spectral(m).spectral.omega.__setitem__((1, 1), np.inf), ir.SPEC_OMEGA),
    ("ls_size", lambda m: setattr(_spectral(m).spectral, "ls", Ref("z")), ir.SPEC_LS),
    ("ls_support", lambda m: setattr(_spectral(m).spectral, "ls", Ref("b0")), ir.SPEC_LS),
    ("ls_const_zero", lambda m: setattr(_spectral(m).spectral, "ls", np.array([0.5, 0.0])), ir.SPEC_LS),
    ("ls_const_size", lambda m: setattr(_spectral(m).spectral, "ls", np.array([0.5, 0.5, 0.5])), ir.SPEC_LS),
    ("amp_support", lambda m: setattr(_spectral(m).spectral, "amplitude", Ref("b0")), ir.SPEC_AMP),
    ("amp_vector", lambda m: setattr(_spectral(m).spectral, "amplitude", Ref("z")), ir.SPEC_AMP),
    ("amp_const", lambda m: setattr(_spectral(m).spectral, "amplitude", -1.0), ir.SPEC_AMP),
]


@pytest.mark.parametrize("what,edit,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_validate_refuses_each_clause(what, edit, msg):
    m = _edit(edit)()
    with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)")):
        m.validate()


def test_inversegamma_prior_rules():
    m = small_model("expquad", 1, "var", "var")
    m.priors[3] = Prior("inversegamma", "ell_log__", (3.0, Ref("sigma_log__")))
    with pytest.raises(ValueError, match="must be a constant"):
        m.validate()
    m.priors[3] = Prior("inversegamma", "ell_log__", (3.0, -1.0))
    with pytest.raises(ValueError, match="InverseGamma needs constant alpha, beta > 0"):
        m.validate()
    m.priors[3] = Prior("inversegamma", "b0", (3.0, 2.0))
    with pytest.raises(ValueError, match="positive support"):
        m.validate()


def _block(low):
    """(Phi [N][M], the spectral block) of the lowered spectral term of small_model."""
    t = low.liks[0]["terms"][1]
    N, M = low.liks[0]["N"], t["n_cols"]
    return t, N, M


def _set_block(k, value):
    def edit(low):
        t, N, M = _block(low)
        c = t["coef"].copy()
        c[N * M + k] = value
        t["coef"] = c
    return edit


def _set_factor(f, value):
    def edit(low):
        t, _, _ = _block(low)
        t["factors"] = [value if j == f else fa for j, fa in enumerate(t["factors"])]
    return edit


def _build_abi():
    return small_model("expquad", 2, "var", "var")


def _build_abi_const():
    return small_model("matern32", 2, "const", "var")


def _phi_nan(low):
    t, _, _ = _block(low)
    c = t["coef"].copy()
    c[3] = np.nan
    t["coef"] = c


ABI_REFUSALS = [
    ("phi_nan", _build_abi, _phi_nan, ir.SPEC_PHI),
    ("z_size", _build_abi, lambda low: _set_factor(0, (_block(low)[0]["factors"][0][0], 3, None))(low), ir.SPEC_PHI),
    ("z_transformed", _build_abi, lambda low: _set_factor(0, (low.n - 3, _block(low)[2], None))(low), ir.SPEC_Z),
    ("cov", _build_abi, _set_block(0, 7.0), ir.SPEC_COV),
    ("dims", _build_abi, _set_block(1, 0.0), ir.SPEC_OMEGA),
    ("omega", _build_abi, lambda low: _set_block(3 + 2 + 1, -1.0)(low), ir.SPEC_OMEGA),
    ("amp_const", _build_abi, lambda low: (_set_factor(1, (0, 0, None))(low), _set_block(2, 0.0)(low)), ir.SPEC_AMP),
    ("amp_var", _build_abi, lambda low: _set_factor(1, (0, 1, None))(low), ir.SPEC_AMP),
    ("ls_var", _build_abi, _set_factor(2, (0, 1, None)), ir.SPEC_LS),
    ("ls_const", _build_abi_const, _set_block(4, -2.0), ir.SPEC_LS),
]


@pytest.mark.parametrize("what,build,edit,msg", ABI_REFUSALS, ids=[r[0] for r in ABI_REFUSALS])
def test_model_create_refuses_malformed_spectral_tables_through_the_c_abi(what, build, edit, msg):
    err = refusal_after_edit(build, edit)
    assert err is not None and msg in err, (what, err)


def test_model_create_refuses_inversegamma_with_a_bad_parameter_through_the_c_abi():
    def edit(low):
        d, v, pars = low.priors[3]
        low.priors[3] = (d, v, [pars[0], (0, -2.0, -1), pars[2]])
    err = refusal_after_edit(_build_abi, edit)
    assert "InverseGamma needs constant alpha, beta > 0" in err


# ---- lowering, Deterministics and the other passes --------------------------------------------------------------------
def test_constant_hyperparameters_lower_to_a_plain_design_term():
    m = small_model("matern52", 2, "const", "const")
    t = ir.lower(m).liks[0]["terms"][1]
    sp = m.likelihoods[0].terms[1].spectral
    s = np.exp(ir.spectral_log_scale(sp.cov, sp.omega, np.asarray(sp.ls), sp.amplitude))
    assert t["n_cols"] == len(s) and len(t["factors"]) == 1
    np.testing.assert_array_equal(t["coef"], m.likelihoods[0].terms[1].coef * s[None, :])


def test_random_hyperparameters_lower_to_the_abi_spectral_term():
    m = small_model("matern32", 2, "iso", "var")
    low = ir.lower(m)
    t, N, M = _block(low)
    off = m.offsets()
    assert t["factors"] == [(off["z"], M, None), (off["eta_log__"], 1, None), (off["ell_log__"], 1, None)]
    blk = t["coef"][N * M :]
    assert blk[0] == ir.COV_FUNCS["matern32"] and blk[1] == 2 and len(blk) == 3 + 2 + M * 2
    np.testing.assert_array_equal(blk[5:].reshape(M, 2), m.likelihoods[0].terms[1].spectral.omega)
    assert low.priors[3][0] == ir.PRIOR_DISTS["inversegamma"][0] == 12


def test_deterministic_f_constant_data_specialise_and_fuse():
    m = ir.hsgp_regression_ir("expquad", n_obs=50, covariates=2)
    q = m.initial_point() + np.random.default_rng(2).uniform(-0.5, 0.5, (3, m.n))
    x = m.constrain(q)
    t = m.likelihoods[0].terms[0]
    f = m.eval_deterministics(x)["f"]
    s = ir.spectral_weights(m, t, x)
    np.testing.assert_allclose(f, (x["f_hsgp_coeffs"] * s) @ t.coef.T, rtol=1e-14)
    cd = m.constant_data()
    np.testing.assert_array_equal(cd["y_omega0"], t.spectral.omega)
    np.testing.assert_array_equal(cd["y_coef0"], t.coef)
    assert ir.specialise(m) is None and ir.specialise(m, extended=True) is None
    fused = ir.fuse_design_columns(m)
    assert fused.likelihoods[0].terms[0].spectral is not None
    np.testing.assert_array_equal(fused.likelihoods[0].terms[0].coef, t.coef)


def test_the_example_builder():
    from oracle import ir_numpy_hsgp

    for kw in (dict(), dict(dims=2), dict(additive=True, cov="matern32"), dict(dist="poisson", covariates=2),
               dict(dist="bernoulli", cov="matern52"), dict(ls="const", amplitude="const")):
        m = ir.hsgp_regression_ir(**kw, n_obs=80)
        m.validate()
        lp, g = ir_numpy_hsgp.make_logp(m)(m.initial_point())
        assert np.isfinite(lp) and np.all(np.isfinite(g)), kw
    assert ir.hsgp_regression_ir(dims=2).var("ell_f_log__").size == 2
    assert ir.hsgp_regression_ir(dims=2).var("f_hsgp_coeffs").size == 144


def test_a_spectral_term_in_logit_psi_is_evaluated():
    """A spectral term may stand in the terms of logit(psi) of a zero-inflated likelihood; its gradient there is right."""
    from oracle import ir_numpy_hsgp

    m = small_model("matern52", 1, "var", "var", N=6)
    t = m.likelihoods[0].terms[1]
    m.likelihoods[0] = Likelihood("zero_inflated_poisson", np.array([0.0, 1.0, 0.0, 3.0, 2.0, 0.0]), [Term([("b0", None)])],
                                  psi=ir.Linear([copy.deepcopy(t)]))
    m.validate()
    f = ir_numpy_hsgp.make_logp(m)
    q = m.initial_point() + np.random.default_rng(3).uniform(-0.5, 0.5, m.n)
    np.testing.assert_allclose(f(q)[1], fd_grad(f, q), rtol=1e-6, atol=1e-6)
    assert ir.lower(m).liks[0]["psi"][0]["n_cols"] == t.coef.shape[1]


def zip_logit_psi_ir():
    """Zero-inflated Poisson counts whose logit(psi) is g0 plus an HSGP term, with b0 + X beta as the count predictor."""
    m = ir.hsgp_regression_ir("expquad", dist="poisson", covariates=2, n_obs=300, seed=91)
    L = m.likelihoods[0]
    rng = np.random.default_rng(92)
    y = np.where(rng.random(len(L.y)) < 0.3, 0.0, L.y)
    m.vars.append(Var("g0", "g0", 1, initial=1.0))
    m.priors.append(Prior("normal", "g0", (0.0, 1.5)))
    m.likelihoods[0] = Likelihood("zero_inflated_poisson", y, L.terms[1:], psi=ir.Linear([Term([("g0", None)]), L.terms[0]]))
    m.name = "hsgp_zip_logit_psi"
    return m


def latent_location_ir(K=40, N=300, seed=93):
    """Group effects a_j ~ Normal(f(x_j), 0.3) whose location is an HSGP over the groups' covariate (a latent factor), and
    y_i ~ Normal(a[g_i], sigma)."""
    rng = np.random.default_rng(seed)
    xg = rng.uniform(0.0, 10.0, K)
    Phi, omega, _, _ = ir.hsgp_basis(xg, 16, c=1.5)
    g = rng.integers(0, K, N).astype(np.int32)
    y = np.sin(xg)[g] + rng.normal(0.0, 0.4, N)
    vars_ = [Var("z", "z", 16), Var("ell_log__", "ell", 1, "log", initial=np.log(2.0)),
             Var("eta_log__", "eta", 1, "log"), Var("a", "a", K), Var("sigma_log__", "sigma", 1, "log")]
    t = Term([("z", None)], coef=Phi, spectral=Spectral("matern32", omega, Ref("ell_log__"), Ref("eta_log__")))
    priors = [Prior("normal", "z", (0.0, 1.0)), Prior("inversegamma", "ell_log__", (4.0, 8.0)),
              Prior("halfnormal", "eta_log__", (1.0,)), Prior("normal", "a", (ir.Linear([t]), 0.3)),
              Prior("halfnormal", "sigma_log__", (1.0,))]
    return ModelIR(name="hsgp_latent_location", vars=vars_, priors=priors,
                   likelihoods=[Likelihood("normal", y, [Term([("a", g)])], sigma=Ref("sigma_log__"))])


def oracle_of(m):
    """ir_numpy_hsgp over the latent-factor oracle when the model has one, else over its default base"""
    from ir_latent_oracle import make_logp as latent_logp
    from oracle import ir_numpy_hsgp

    return ir_numpy_hsgp.make_logp(m, latent_logp if any(ir.is_latent(p) for p in m.priors) else None)


def test_a_spectral_term_in_a_latent_location_is_evaluated():
    """A spectral term may stand in a Linear prior location; the oracle's gradient there is right, and it lowers to a
    spectral term of the latent factor."""
    m = latent_location_ir(K=8, N=30)
    f = oracle_of(m)
    q = m.initial_point() + np.random.default_rng(3).uniform(-0.5, 0.5, m.n)
    np.testing.assert_allclose(f(q)[1], fd_grad(f, q), rtol=1e-6, atol=1e-6)
    latent = ir.lower(m).liks[1]
    assert latent["y_var"] > 0 and latent["terms"][0]["n_cols"] == 16 and len(latent["terms"][0]["factors"]) == 3


def test_the_zero_inflated_builder_is_evaluated():
    m = zip_logit_psi_ir()
    f = oracle_of(m)
    q = m.initial_point() + np.random.default_rng(4).uniform(-0.3, 0.3, m.n)
    np.testing.assert_allclose(f(q)[1], fd_grad(f, q), rtol=1e-6, atol=1e-6 * max(1.0, np.max(np.abs(f(q)[1]))))


# ---- GPU ---------------------------------------------------------------------------------------------------------------
BUILDERS = {
    "zip_logit_psi": zip_logit_psi_ir,
    "latent_location": latent_location_ir,
    "expquad_1d": lambda: ir.hsgp_regression_ir("expquad"),
    "matern52_2d_ard": lambda: ir.hsgp_regression_ir("matern52", dims=2),
    "matern32_additive": lambda: ir.hsgp_regression_ir("matern32", additive=True),
    "poisson_covariates": lambda: ir.hsgp_regression_ir("expquad", dist="poisson", covariates=2),
    "bernoulli_matern52": lambda: ir.hsgp_regression_ir("matern52", dist="bernoulli"),
    "const_ls": lambda: ir.hsgp_regression_ir("expquad", ls="const"),
    "expquad_2d_cta": lambda: ir.hsgp_regression_ir("expquad", dims=2, m=18),
}


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(CASES))
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid):
    from oracle import ir_numpy_hsgp
    from pymc_b200 import engine

    m = small_model(*CASES[cid])
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = ir_numpy_hsgp.make_logp(m)
    Q = case_points(m)
    lp_mp, g_mp = mp_reference(m, Q)
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    for team, (lp, g) in logp_at_both_team_shapes(cm, Q).items():
        assert np.all(np.isfinite(lp)) and np.all(np.isfinite(g)), (cid, team)
        assert_close(lp, g, lp_mp, g_mp, 1e-12, (cid, team))
        assert_close(lp, g, lo, go, 1e-12, (cid, team, "oracle"))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_device_function_matches_the_oracle_on_the_builders(name):
    from pymc_b200 import engine

    m = BUILDERS[name]()
    cm = engine.CompiledModel(m)
    assert cm.spec.name == "ir" and (m.n > 256) == name.endswith("cta")
    f = oracle_of(m)
    Q = m.initial_point() + np.random.default_rng(0).uniform(-1.0, 1.0, (9, m.n))
    lo, go = np.array([f(q)[0] for q in Q]), np.array([f(q)[1] for q in Q])
    for team, (lp, g) in logp_at_both_team_shapes(cm, Q).items():
        assert_close(lp, g, lo, go, 1e-12, (name, team))


def scipy_pointwise(m, q):
    from oracle import ir_numpy_hsgp

    f = ir_numpy_hsgp.make_logp(m)
    L = m.likelihoods[0]
    out = np.empty(q.shape[:-1] + (len(L.y),))
    for ix in np.ndindex(*q.shape[:-1]):
        x, _ = f.constrained(q[ix])
        qe, _ = f.extended(x, q[ix])
        eta = sum(qe[us] for _, us in f.design)
        for t in L.terms:
            if not ir.is_design(t):
                eta = eta + x[m.offsets()[t.factors[0][0]]]
        if L.dist == "normal":
            out[ix] = stats.norm.logpdf(L.y, eta, x[m.offsets()["sigma_log__"]])
        elif L.dist == "poisson_log":
            out[ix] = stats.poisson.logpmf(L.y, np.exp(eta))
        else:
            out[ix] = stats.bernoulli.logpmf(L.y, 1.0 / (1.0 + np.exp(-eta)))
    return out


@pytest.mark.gpu
def test_pointwise_log_likelihood_matches_scipy():
    from pymc_b200 import engine

    for name in ("expquad_1d", "matern52_2d_ard", "poisson_covariates", "bernoulli_matern52"):
        m = BUILDERS[name]()
        cm = engine.CompiledModel(m, specialise=False)
        q = m.initial_point() + np.random.default_rng(4).uniform(-0.5, 0.5, (2, 3, m.n))
        np.testing.assert_allclose(cm.pointwise_loglik(q), scipy_pointwise(m, q), rtol=1e-11, atol=1e-11, err_msg=name)


@pytest.mark.gpu
@pytest.mark.parametrize("name,eps", [("expquad_1d", 0.05), ("matern52_2d_ard", 0.05), ("matern32_additive", 0.05),
                                      ("poisson_covariates", 0.03), ("bernoulli_matern52", 0.1), ("const_ls", 0.05),
                                      ("expquad_2d_cta", 0.03), ("zip_logit_psi", 0.03), ("latent_location", 0.05)])
def test_fixed_step_nuts_matches_the_oracle_sampler(name, eps):
    m = BUILDERS[name]()
    fixed_step_against_oracle(m, oracle_of(m), eps, C=2, T=8)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle():
    from oracle import ir_numpy_hsgp

    m = ir.hsgp_regression_ir("expquad", n_obs=150, m=16)
    fixed_step_against_oracle(m, ir_numpy_hsgp.make_logp(m), 0.1, dense_cov=random_dense_cov(m.n, 2, 0.02, 0.05, 12),
                              C=2, T=8)


@pytest.mark.gpu
def test_adaptive_run_with_random_lengthscale_and_amplitude_matches_the_oracle_posterior():
    from oracle import ir_numpy_hsgp

    m = ir.hsgp_regression_ir("expquad", n_obs=120, m=16)
    adaptive_against_oracle(m, ir_numpy_hsgp.make_logp(m), chain_seed=23, spread=0.5, philox_seed=5, oracle_seed=200,
                            se_bound=5.0, max_divergence=0.02)


@pytest.mark.gpu
def test_sample_returns_f_in_the_posterior():
    import pymc_b200

    m = ir.hsgp_regression_ir("matern52", n_obs=100, m=16)
    res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, compute_convergence_checks=False)
    f = np.asarray(res.posterior["f"])
    assert f.shape == (4, 20, 100) and np.all(np.isfinite(f))
    x = {k: np.asarray(res.posterior[k]) for k in ("f_hsgp_coeffs", "ell_f", "eta_f")}
    np.testing.assert_allclose(f, m.eval_deterministics(x)["f"], rtol=1e-12, atol=1e-12)
