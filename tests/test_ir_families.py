"""Binomial (logit link), negative-binomial (log link, random dispersion) and Gamma (log link, random shape) likelihoods of the
IR: the NumPy restatement (oracle/ir_numpy_families.py) against scipy.stats, central differences and the reference's own
known answers; validation and lowering; the stored reference golden replayed by the oracle NUTS.  The generic device
function is checked against the restatement in the `gpu`-marked tests at the bottom."""
import ctypes

import numpy as np
import pytest
from scipy import stats

from b200_helpers import adaptive_against_oracle, fd_grad, fixed_step_against_oracle, random_dense_cov, refusal_after_edit

from pymc_b200 import _lib, ir


def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def _data(dist, eta, rng):
    if dist == "binomial_logit":
        n = rng.integers(0, 30, len(eta)).astype(float)
        return rng.binomial(n.astype(int), _sigmoid(eta)).astype(float), n
    if dist == "negative_binomial_log":
        return rng.negative_binomial(2.0, 2.0 / (np.exp(eta) + 2.0)).astype(float), None
    return rng.gamma(2.0, np.exp(eta) / 2.0), None


def _scipy_loglik(dist, y, eta, a, n):
    if dist == "binomial_logit":
        return stats.binom.logpmf(y, n, _sigmoid(eta))
    mu = np.exp(eta)
    if dist == "negative_binomial_log":
        return stats.nbinom.logpmf(y, a, a / (mu + a))
    return stats.gamma.logpdf(y, a, scale=mu / a)


FAMILY_CASES = [("binomial_logit", "array"), ("binomial_logit", "scalar"), ("negative_binomial_log", "const"),
                ("negative_binomial_log", "ref"), ("gamma_log", "const"), ("gamma_log", "ref")]


def _family_model(dist, kind, seed=0):
    """b0 + b1 x under the family; a random dispersion is alpha ~ Exponential(1) on the log scale."""
    rng = np.random.default_rng(seed)
    N = 50
    x = rng.standard_normal(N)
    eta0 = 0.8 + 0.6 * x
    y, n = _data(dist, eta0, rng)
    vars_ = [ir.Var("b0", "b0", 1), ir.Var("b1", "b1", 1)]
    priors = [ir.Prior("normal", "b0", (0.0, 2.0)), ir.Prior("normal", "b1", (0.0, 1.0))]
    kw = {}
    if dist == "binomial_logit":
        if kind == "scalar":
            n = np.full(N, 30.0)
            y = np.minimum(y, 30.0)
            kw["trials"] = 30.0
        else:
            kw["trials"] = n
    elif kind == "ref":
        vars_.append(ir.Var("alpha_log__", "alpha", 1, "log", initial=np.log(2.0)))
        priors.append(ir.Prior("exponential", "alpha_log__", (1.0,)))
        kw["alpha"] = ir.Ref("alpha_log__")
    else:
        kw["alpha"] = 2.5
    terms = [ir.Term([("b0", None)]), ir.Term([("b1", None)], coef=x)]
    return ir.ModelIR(vars=vars_, priors=priors, likelihoods=[ir.Likelihood(dist, y, terms, **kw)]), x, n


@pytest.mark.parametrize("dist,kind", FAMILY_CASES, ids=[f"{d}-{k}" for d, k in FAMILY_CASES])
def test_family_densities_against_scipy_and_central_differences(dist, kind):
    """logp = priors + Jacobians (oracle/ir_numpy.py) + the scipy.stats log-pmf / log-pdf of every observation; the gradient,
    including d/d alpha through digamma for a random dispersion, matches central differences."""
    import dataclasses

    from oracle import ir_numpy, ir_numpy_families

    m, x, n = _family_model(dist, kind)
    f = ir_numpy_families.make_logp(m)
    rest = ir_numpy.make_logp(dataclasses.replace(m, likelihoods=[]))
    L = m.likelihoods[0]
    rng = np.random.default_rng(1)
    for _ in range(4):
        q = m.initial_point() + rng.uniform(-0.7, 0.7, m.n)
        lp, g = f(q)
        c = m.constrain(q)
        a = c["alpha"] if kind == "ref" else (L.alpha if L.alpha is not None else None)
        want = rest(q)[0] + np.sum(_scipy_loglik(dist, L.y, c["b0"] + c["b1"] * x, a, n))
        assert abs(lp - want) <= 1e-12 * abs(want)
        assert np.max(np.abs(fd_grad(f, q) - g)) <= 5e-6 * max(1.0, np.max(np.abs(g)))


def test_family_gradients_through_a_hierarchical_predictor_by_central_differences():
    """The families under the bilinear / indexed predictor of test_ir.py's hierarchical case, with a random dispersion
    that also parametrises a prior."""
    from oracle import ir_numpy_families

    rng = np.random.default_rng(3)
    N, G = 40, 5
    g = rng.integers(0, G, N).astype(np.int32)
    xcov = rng.standard_normal(N)
    vars_ = [ir.Var("m", "m", 1), ir.Var("s_log__", "s", 1, "log"), ir.Var("a", "a", G), ir.Var("b", "b", 1),
             ir.Var("alpha_log__", "alpha", 1, "log")]
    pri = [ir.Prior("normal", "m", (0.0, 2.0)), ir.Prior("halfnormal", "s_log__", (1.0,)),
           ir.Prior("normal", "a", (ir.Ref("m"), ir.Ref("s_log__"))), ir.Prior("cauchy", "b", (0.0, ir.Ref("s_log__"))),
           ir.Prior("halfnormal", "alpha_log__", (ir.Ref("s_log__"),))]
    terms = [ir.Term([("a", g)]), ir.Term([("b", None)], coef=xcov), ir.Term([("s_log__", None), ("a", g), ("b", None)], coef=0.1)]
    for dist, y, kw in [("binomial_logit", rng.integers(0, 6, N).astype(float), dict(trials=np.full(N, 8.0))),
                        ("negative_binomial_log", rng.poisson(3.0, N).astype(float), dict(alpha=ir.Ref("alpha_log__"))),
                        ("gamma_log", rng.gamma(2.0, 1.0, N), dict(alpha=ir.Ref("alpha_log__")))]:
        m = ir.ModelIR(vars=vars_, priors=pri, likelihoods=[ir.Likelihood(dist, y, terms, **kw)])
        f = ir_numpy_families.make_logp(m)
        q = rng.uniform(-0.8, 0.8, m.n)
        lp, gr = f(q)
        assert np.isfinite(lp)
        assert np.max(np.abs(fd_grad(f, q) - gr)) <= 5e-6 * max(1.0, np.max(np.abs(gr))), dist


def _one_obs_nb(y, alpha):
    return ir.ModelIR(vars=[ir.Var("eta", "eta", 1)],
                      likelihoods=[ir.Likelihood("negative_binomial_log", np.array([float(y)]), [ir.Term([("eta", None)])],
                                                 alpha=alpha)])


def test_negative_binomial_reference_known_answers_and_stability():
    """tests/distributions/test_discrete.py of the reference: test_negative_binomial_logp_large_n (mu = 5, alpha = 1e12,
    y = 3: the Poisson limit) and test_negative_binomial_logp_stable_when_p_underflows (alpha = 2, y = 3, p = sigmoid(-800)).
    Where mu = exp(eta) overflows (an xfail of the reference) the log-sum-exp form stays finite."""
    from oracle import ir_numpy_families

    lp, g = ir_numpy_families.make_logp(_one_obs_nb(3, 1e12))(np.array([np.log(5.0)]))
    assert abs(lp - -1.9634457319257537) <= 1e-12 * 2.0 and abs(g[0] - (3.0 - 5.0)) <= 1e-12
    f = ir_numpy_families.make_logp(_one_obs_nb(3, 2.0))
    lp, g = f(np.array([800.0 + np.log(2.0)]))
    assert abs(lp - -1598.6137056388802) <= 1e-12 * 1598.6137056388802 and abs(g[0] - -2.0) <= 1e-12
    for eta in (1000.0, -1000.0):
        lp, g = f(np.array([eta]))
        assert np.isfinite(lp) and np.all(np.isfinite(g))
    m = ir.ModelIR(vars=[ir.Var("eta", "eta", 1), ir.Var("alpha_log__", "alpha", 1, "log")],
                   likelihoods=[ir.Likelihood("negative_binomial_log", np.array([3.0, 0.0]), [ir.Term([("eta", None)])],
                                              alpha=ir.Ref("alpha_log__"))])
    lp, g = ir_numpy_families.make_logp(m)(np.array([1000.0, np.log(2.0)]))
    assert np.isfinite(lp) and np.all(np.isfinite(g))


def test_validation_rejects_out_of_support_data_and_parameters():
    v = [ir.Var("b", "b", 1), ir.Var("s_log__", "s", 1, "log"), ir.Var("u", "u", 1), ir.Var("p_interval__", "p", 1, "interval", (-1.0, 1.0)),
         ir.Var("v", "v", 2, "log")]
    t = [ir.Term([("b", None)])]

    def bad(*liks):
        for L in liks:
            with pytest.raises(ValueError):
                ir.ModelIR(vars=v, likelihoods=[L]).validate()

    y3 = np.array([0.0, 2.0, 3.0])
    bad(ir.Likelihood("binomial_logit", y3, t, trials=2.0),                         # y > n
        ir.Likelihood("binomial_logit", np.array([0.5, 1.0, 1.0]), t, trials=3.0),  # y not an integer
        ir.Likelihood("binomial_logit", np.array([-1.0, 1.0, 1.0]), t, trials=3.0),  # y < 0
        ir.Likelihood("binomial_logit", y3, t, trials=np.array([3.0, 3.0, -3.0])),  # trials < 0
        ir.Likelihood("binomial_logit", y3, t, trials=3.5),                         # trials not an integer
        ir.Likelihood("binomial_logit", y3, t, trials=np.array([3.0, 3.0])),        # length
        ir.Likelihood("binomial_logit", y3, t),                                     # trials missing
        ir.Likelihood("binomial_logit", y3, t, trials=ir.Ref("s_log__")),            # trials must be constant
        ir.Likelihood("negative_binomial_log", np.array([-1.0, 2.0]), t, alpha=1.0),  # y < 0
        ir.Likelihood("negative_binomial_log", np.array([1.5, 2.0]), t, alpha=1.0),  # y not an integer
        ir.Likelihood("negative_binomial_log", y3, t, alpha=0.0),                  # alpha <= 0
        ir.Likelihood("negative_binomial_log", y3, t),                              # alpha missing
        ir.Likelihood("negative_binomial_log", y3, t, alpha=ir.Ref("u")),           # no positive support
        ir.Likelihood("negative_binomial_log", y3, t, alpha=ir.Ref("p_interval__")),  # interval reaching below 0
        ir.Likelihood("negative_binomial_log", y3, t, alpha=ir.Ref("v")),           # vector alpha
        ir.Likelihood("gamma_log", np.array([0.0, 1.0]), t, alpha=1.0),             # y <= 0
        ir.Likelihood("gamma_log", np.array([-2.0, 1.0]), t, alpha=1.0),
        ir.Likelihood("gamma_log", np.array([2.0, 1.0]), t, alpha=-1.0),            # alpha <= 0
        ir.Likelihood("gamma_log", np.array([2.0, 1.0]), t, alpha=ir.Ref("v")),     # vector alpha
        ir.Likelihood("gamma_log", np.array([2.0, 1.0]), t, alpha=1.0, sigma=1.0),  # no sigma
        ir.Likelihood("poisson_log", y3, t, alpha=1.0))                             # alpha of another family
    for L in (ir.Likelihood("binomial_logit", y3, t, trials=3.0), ir.Likelihood("negative_binomial_log", y3, t, alpha=ir.Ref("s_log__")),
              ir.Likelihood("gamma_log", np.array([2.0, 1.0]), t, alpha=ir.Ref("s_log__"))):
        ir.ModelIR(vars=v, likelihoods=[L]).validate()
    ok = [ir.Var("b", "b", 1), ir.Var("a_interval__", "a", 1, "interval", (0.0, 5.0))]
    ir.ModelIR(vars=ok, likelihoods=[ir.Likelihood("gamma_log", np.array([2.0]), t, alpha=ir.Ref("a_interval__"))]).validate()


def test_validation_still_checks_ar1_without_likelihoods_and_rejects_non_finite_parameters():
    """The AR(1) checks of validate() run for a model with no likelihood; infinite trials or alpha are refused."""
    with pytest.raises(ValueError, match="two steps"):
        ir.ModelIR(vars=[ir.Var("h", "h", 1), ir.Var("phi", "phi", 2)], ar1=[ir.AR1("h", ir.Ref("phi"), 1.0)]).validate()
    with pytest.raises(ValueError, match="scalar"):
        ir.ModelIR(vars=[ir.Var("h", "h", 5), ir.Var("phi", "phi", 2)], ar1=[ir.AR1("h", ir.Ref("phi"), 1.0)]).validate()
    t = [ir.Term([("b", None)])]
    v = [ir.Var("b", "b", 1)]
    for L in (ir.Likelihood("binomial_logit", np.array([1.0]), t, trials=np.inf),
              ir.Likelihood("negative_binomial_log", np.array([1.0]), t, alpha=np.inf),
              ir.Likelihood("gamma_log", np.array([1.0]), t, alpha=np.inf),
              ir.Likelihood("gamma_log", np.array([np.inf]), t, alpha=1.0)):
        with pytest.raises(ValueError):
            ir.ModelIR(vars=v, likelihoods=[L]).validate()


def test_lowering_puts_trials_and_alpha_in_the_parameter_slot():
    def lik0(m):
        c_ir, keep = _lib.build_ir(ir.lower(m))
        return ctypes.cast(c_ir.liks, ctypes.POINTER(_lib.IrLik))[0], keep

    m = ir.negative_binomial_ir(n_obs=60, n_groups=4, seed=2)
    lik, keep = lik0(m)
    assert lik.dist == 6 and lik.N == 60 and lik.n_terms == 4
    assert lik.sigma_kind == ir.SIGMA_REF and lik.sigma.kind == 1 and lik.sigma.ref == m.offsets()["alpha_log__"] == m.n - 1
    lik, keep = lik0(ir.negative_binomial_ir(n_obs=60, n_groups=4, seed=2, alpha=3.5))
    assert lik.sigma_kind == ir.SIGMA_CONST and lik.sigma.kind == 0 and lik.sigma.value == 3.5 and not lik.sigma_obs
    g = ir.gamma_regression_ir(n_obs=30)
    lik, keep = lik0(g)
    assert lik.dist == 7 and lik.sigma_kind == ir.SIGMA_REF and lik.sigma.ref == g.offsets()["alpha_log__"]
    b = ir.binomial_logit_ir(n_obs=40)
    lik, keep = lik0(b)
    trials = np.ctypeslib.as_array(ctypes.cast(lik.sigma_obs, ctypes.POINTER(ctypes.c_double)), (40,))
    assert lik.dist == 5 and lik.sigma_kind == ir.SIGMA_OBS and np.array_equal(trials, b.likelihoods[0].trials)
    b.likelihoods[0].trials = 40.0
    lik, keep = lik0(b)
    assert lik.sigma_kind == ir.SIGMA_CONST and lik.sigma.value == 40.0 and not lik.sigma_obs


def test_builders_stay_on_the_generic_path_and_record_their_data():
    for m in (ir.binomial_logit_ir(), ir.negative_binomial_ir(), ir.negative_binomial_ir(alpha=2.0), ir.gamma_regression_ir(),
              ir.gamma_regression_ir(alpha=2.0)):
        m.validate()
        assert ir.specialise(m) is None and ir.specialise(m, extended=True) is None
    b = ir.binomial_logit_ir()
    assert np.array_equal(b.constant_data()["y_trials"], b.likelihoods[0].trials)
    assert "y_trials" not in ir.negative_binomial_ir().constant_data()
    assert ir.negative_binomial_ir(n_groups=400, n_obs=2000).n > 256 and ir.negative_binomial_ir().n <= 256


def test_oracle_nuts_reproduces_the_negative_binomial_golden(golden):
    """tests/golden/negbin_fixed.npz: the reference's own NUTS (oracle/make_golden_families.py) on the NumPy density of the
    negative-binomial regression with a random alpha; the oracle must reproduce whole chains."""
    from oracle import ir_numpy_families, nuts_numpy
    from test_oracle_golden import _gen_from_state

    d = golden("negbin_fixed")
    m = ir.negative_binomial_ir()
    f = ir_numpy_families.make_logp(m)
    for c in range(len(d["seeds"])):
        o = nuts_numpy.Oracle(f, nuts_numpy.DiagMass(d["var"][c]), adapt_step_size=False)
        o.da = nuts_numpy.DualAveraging(float(d["used_eps"][c][0]))
        o.rng, o.tune = _gen_from_state(d["pre_rng"][c][0]), False
        qs, st = o.run(d["q0"][c], 0, int(d["draws"]), z=d["z"][c])
        assert np.array_equal(st["tree_size"], d["stat_tree_size"][c])
        assert np.array_equal(st["index_in_trajectory"], d["stat_index_in_trajectory"][c])
        assert np.array_equal(qs, d["draws_q"][c])
        assert np.array_equal(st["energy"], d["stat_energy"][c])


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
FAMILY_MODELS = {
    "binomial": ir.binomial_logit_ir,                                                     # n = 13: chain = warp
    "binomial_scalar_trials": lambda: _scalar_trials(ir.binomial_logit_ir()),
    "binomial_cta": lambda: ir.binomial_logit_ir(n_obs=1500, n_groups=300, seed=5),      # n = 303: chain = CTA
    "negbin": ir.negative_binomial_ir,
    "negbin_const": lambda: ir.negative_binomial_ir(alpha=2.5),
    "negbin_cta": lambda: ir.negative_binomial_ir(n_obs=2000, n_groups=400, seed=7),     # n = 405
    "negbin_cta_const": lambda: ir.negative_binomial_ir(n_obs=2000, n_groups=400, seed=7, alpha=2.5),
    "gamma": ir.gamma_regression_ir,
    "gamma_const": lambda: ir.gamma_regression_ir(alpha=3.0),
    "gamma_cta": lambda: ir.gamma_regression_ir(n_obs=1200, n_features=300, seed=9),     # n = 302
    "gamma_cta_const": lambda: ir.gamma_regression_ir(n_obs=1200, n_features=300, seed=9, alpha=3.0),
}


def _scalar_trials(m):
    L = m.likelihoods[0]
    L.y = np.minimum(L.y, 20.0)
    L.trials = 20.0
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FAMILY_MODELS))
def test_device_function_matches_the_family_oracle(name):
    from oracle import ir_numpy_families
    from pymc_b200 import engine

    m = FAMILY_MODELS[name]()
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = ir_numpy_families.make_logp(m)
    rng = np.random.default_rng(0)
    Q = m.initial_point() + rng.uniform(-1.0, 1.0, (23, m.n))
    lp, g = cm.logp_dlogp(Q)
    lo = np.array([f(q)[0] for q in Q])
    go = np.array([f(q)[1] for q in Q])
    assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12
    assert np.max(np.abs(g - go) / np.max(np.abs(go), axis=1, keepdims=True)) <= 1e-12
    lp2, g2 = cm.logp_dlogp(Q)  # deterministic: no atomics, fixed-order sums over the distinct-value table
    assert np.array_equal(lp, lp2) and np.array_equal(g, g2)


@pytest.mark.gpu
def test_device_negative_binomial_known_answers_and_extreme_predictors():
    from oracle import ir_numpy_families
    from pymc_b200 import engine

    lp, g = engine.CompiledModel(_one_obs_nb(3, 1e12), specialise=False).logp_dlogp(np.array([[np.log(5.0)]]))
    assert abs(lp[0] - -1.9634457319257537) <= 1e-12 * 2.0
    cm = engine.CompiledModel(_one_obs_nb(3, 2.0), specialise=False)
    lp, g = cm.logp_dlogp(np.array([[800.0 + np.log(2.0)], [1000.0], [-1000.0]]))
    assert abs(lp[0] - -1598.6137056388802) <= 1e-12 * 1598.6137056388802 and abs(g[0, 0] - -2.0) <= 1e-12
    assert np.all(np.isfinite(lp)) and np.all(np.isfinite(g))
    m = ir.ModelIR(vars=[ir.Var("eta", "eta", 1), ir.Var("alpha_log__", "alpha", 1, "log")],
                   likelihoods=[ir.Likelihood("negative_binomial_log", np.array([3.0, 0.0, 7.0, 3.0]), [ir.Term([("eta", None)])],
                                              alpha=ir.Ref("alpha_log__"))])
    Q = np.array([[1000.0, np.log(2.0)], [-30.0, 3.0], [2.0, np.log(2e10)], [1.0, -4.0]])
    lp, g = engine.CompiledModel(m, specialise=False).logp_dlogp(Q)
    f = ir_numpy_families.make_logp(m)
    for k, q in enumerate(Q):
        lo, go = f(q)
        assert np.isfinite(lp[k]) and abs(lp[k] - lo) <= 1e-12 * abs(lo)
        assert np.max(np.abs(g[k] - go)) <= 1e-12 * max(1.0, np.max(np.abs(go)))


@pytest.mark.gpu
def test_negative_binomial_reproduces_the_reference_golden_on_the_generic_function(golden):
    """negbin_fixed.npz (the reference NUTS on the model's NumPy density): identical tree statistics for every draw and
    positions to 1e-9 on the generic device function."""
    from b200_helpers import discrete_equal, gpu_free_run
    from pymc_b200 import engine

    d = golden("negbin_fixed")
    cm = engine.CompiledModel(ir.negative_binomial_ir(), specialise=False)
    res, _ = gpu_free_run(cm, d, "negbin_fixed")
    for c in range(len(d["seeds"])):
        st = {k: v[c] for k, v in res.stats.items()}
        assert discrete_equal(st, d, c).all(), c
        assert np.max(np.abs(res.draws[c] - d["draws_q"][c])) <= 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("name,eps", [("binomial", 0.05), ("gamma", 0.05), ("negbin_cta", 0.02)])
def test_fixed_step_nuts_matches_the_oracle_sampler(name, eps):
    from oracle import ir_numpy_families

    m = FAMILY_MODELS[name]()
    fixed_step_against_oracle(m, ir_numpy_families.make_logp(m), eps)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle_on_the_negative_binomial_model():
    from oracle import ir_numpy_families

    m = ir.negative_binomial_ir()
    fixed_step_against_oracle(m, ir_numpy_families.make_logp(m), 0.3, dense_cov=random_dense_cov(m.n, 3, 0.04, 0.05, 12),
                              C=2, T=10)


@pytest.mark.gpu
def test_adaptive_negative_binomial_run_matches_the_oracle_posterior():
    """64 device chains against 8 oracle chains (NUTS with diagonal mass adaptation) on the hierarchical negative-binomial
    regression with a random alpha: posterior means within 5 SE, standard deviations within 25 %, few divergences."""
    from oracle import ir_numpy_families

    m = ir.negative_binomial_ir()
    adaptive_against_oracle(m, ir_numpy_families.make_logp(m), specialise=True, chain_seed=21, spread=1, philox_seed=3,
                            oracle_seed=100, se_bound=5.0, max_divergence=0.02)


def _scipy_pointwise(m, q):
    """log p(y_i | draw) per observation from scipy.stats, for the builders' linear predictors."""
    from oracle import ir_numpy_families

    L = m.likelihoods[0]
    c = m.constrain(q)
    off = m.offsets()
    out = np.empty(q.shape[:-1] + (len(L.y),))
    for ix in np.ndindex(*q.shape[:-1]):
        x = q[ix].copy()
        for v in m.vars:
            x[off[v.name] : off[v.name] + v.size] = np.ravel(c[v.rv_name][ix])
        eta = np.zeros(len(L.y))
        for t in L.terms:
            term = np.ones(len(L.y)) if t.coef is None else np.asarray(t.coef, dtype=np.float64)
            for vn, idx in t.factors:
                v = m.var(vn)
                xv = x[off[v.name] : off[v.name] + v.size]
                term = term * (xv[idx] if idx is not None else xv)
            eta += term
        a = float(np.ravel(c["alpha"][ix])[0]) if "alpha" in c else L.alpha
        out[ix] = _scipy_loglik(L.dist, L.y, eta, a, L.trials)
        assert np.allclose(out[ix], ir_numpy_families.family_loglik(L, eta, a), rtol=1e-12, atol=1e-12)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["binomial", "binomial_scalar_trials", "negbin", "negbin_const", "gamma", "gamma_const"])
def test_pointwise_log_likelihood_matches_scipy(name):
    from pymc_b200 import engine

    m = FAMILY_MODELS[name]()
    cm = engine.CompiledModel(m, specialise=False)
    q = m.initial_point() + np.random.default_rng(4).uniform(-0.5, 0.5, (2, 5, m.n))
    ll = cm.pointwise_loglik(q)
    assert ll.shape == (2, 5, len(m.likelihoods[0].y))
    np.testing.assert_allclose(ll, _scipy_pointwise(m, q), rtol=1e-12, atol=1e-12)


@pytest.mark.gpu
def test_sampler_records_the_log_likelihood_group_for_the_families():
    import pymc_b200

    for m in (ir.negative_binomial_ir(), ir.gamma_regression_ir(), ir.binomial_logit_ir()):
        res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, keep_untransformed=True,
                                         idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
        ll = res.log_likelihood["y"]
        assert ll.shape == (4, 20, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, _scipy_pointwise(m, res.unconstrained), rtol=1e-12, atol=1e-12)
        if "alpha" in res.posterior:
            assert np.all(res.posterior["alpha"] > 0)
        if m.likelihoods[0].trials is not None:
            assert np.array_equal(res.constant_data["y_trials"], m.likelihoods[0].trials)


def test_model_create_rejects_out_of_support_tables_through_the_c_abi():
    """prepare_ir checks what validate() checks, for callers of the C ABI that bypass the Python front end."""
    def setter(**kw):
        def f(low):
            L = low.liks[0]
            for k, v in kw.items():
                if k == "y0":
                    L["y"] = L["y"].copy()
                    L["y"][0] = v
                elif k == "n0":
                    L["sigma_obs"] = L["sigma_obs"].copy()
                    L["sigma_obs"][0] = v
                else:
                    L[k] = v
        return f

    b, nb, ga = ir.binomial_logit_ir, lambda: ir.negative_binomial_ir(alpha=2.0), lambda: ir.gamma_regression_ir(alpha=2.0)
    nb_ref, ga_ref = ir.negative_binomial_ir, ir.gamma_regression_ir
    for builder, edit, msg in [
        (b, setter(y0=1e6), "Binomial y"),                     # y > n
        (b, setter(y0=0.5), "Binomial y"),                     # not an integer
        (b, setter(n0=-1.0), "Binomial trials"),               # trials < 0
        (b, setter(n0=2.5), "Binomial trials"),                # not an integer
        (b, setter(n0=np.inf), "Binomial trials"),             # infinite
        (b, setter(sigma_kind=ir.SIGMA_NONE), "Binomial trials"),
        (nb, setter(y0=-1.0), "NegativeBinomial y"),
        (nb, setter(y0=1.5), "NegativeBinomial y"),
        (nb, setter(sigma_value=0.0), "NegativeBinomial alpha"),
        (nb, setter(sigma_value=np.inf), "NegativeBinomial alpha"),
        (ga, setter(y0=0.0), "Gamma y"),
        (ga, setter(sigma_value=-1.0), "Gamma alpha"),
        (ga, setter(sigma_value=np.inf), "Gamma alpha"),
        (nb_ref, setter(sigma_ref=0), "positive support"),     # alpha pointing at mu_a (no transform)
        (ga_ref, setter(sigma_ref=0), "positive support"),     # alpha pointing at b0
    ]:
        err = refusal_after_edit(builder, edit)
        assert err is not None and msg in err, (msg, err)
