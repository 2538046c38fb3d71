"""ModelSpec IR: the NumPy evaluation (oracle/ir_numpy.py) against the hand-derived restatements and scipy.stats, the
pattern matcher behind the hand-specialised kernels, and the lowering to the C ABI tables.  GPU parity of the generic
device function is in the `gpu`-marked tests at the bottom."""
import ctypes

import numpy as np
import pytest
from scipy import stats

from b200_helpers import adaptive_against_oracle, fd_grad, fixed_step_against_oracle

from pymc_b200 import _lib, ir, models


@pytest.mark.parametrize("name", ["eight_schools", "radon", "stochvol"])
def test_ir_forms_of_the_baseline_models_equal_the_hand_derived_oracle(name):
    from oracle import ir_numpy, logp_numpy

    irm, spec = {"eight_schools": (ir.eight_schools_ir(), models.eight_schools()),
                 "radon": (ir.radon_ir(), models.radon()),
                 "stochvol": (ir.stochvol_ir(T=150), models.stochvol(T=150))}[name]
    f, g = ir_numpy.make_logp(irm), logp_numpy.make_logp(spec)
    assert irm.n == spec.n and np.array_equal(irm.initial_point(), spec.initial_point())
    assert [v.name for v in irm.vars] == [v.name for v in spec.vars]
    rng = np.random.default_rng(0)
    for _ in range(5):
        q = spec.initial_point() + rng.uniform(-1.5, 1.5, spec.n)
        (a, ga), (b, gb) = f(q), g(q)
        assert abs(a - b) <= 1e-13 * abs(b)
        assert np.max(np.abs(ga - gb)) <= 1e-13 * np.max(np.abs(gb))
    q = rng.uniform(-1, 1, (3, spec.n))
    c1, c2 = irm.constrain(q), spec.constrain(q)
    assert set(c1) == set(c2) and all(np.allclose(c1[k], c2[k], rtol=1e-15) for k in c1)


PRIOR_CASES = [
    ("normal", (0.3, 1.7), None, lambda x: stats.norm(0.3, 1.7).logpdf(x)),
    ("halfnormal", (1.3,), "log", lambda x: stats.halfnorm(scale=1.3).logpdf(x)),
    ("cauchy", (-0.2, 2.0), None, lambda x: stats.cauchy(-0.2, 2.0).logpdf(x)),
    ("halfcauchy", (2.5,), "log", lambda x: stats.halfcauchy(scale=2.5).logpdf(x)),
    ("exponential", (3.0,), "log", lambda x: stats.expon(scale=1 / 3.0).logpdf(x)),
    ("studentt", (4.0, 0.5, 1.2), None, lambda x: stats.t(4.0, 0.5, 1.2).logpdf(x)),
    ("uniform", (-1.0, 3.0), "interval", lambda x: stats.uniform(-1.0, 4.0).logpdf(x)),
    ("gamma", (2.5, 1.5), "log", lambda x: stats.gamma(2.5, scale=1 / 1.5).logpdf(x)),
    ("beta", (2.0, 3.5), "interval01", lambda x: stats.beta(2.0, 3.5).logpdf(x)),
    ("lognormal", (0.2, 0.7), "log", lambda x: stats.lognorm(0.7, scale=np.exp(0.2)).logpdf(x)),
]


@pytest.mark.parametrize("dist,params,tr,ref", PRIOR_CASES, ids=[c[0] for c in PRIOR_CASES])
def test_prior_densities_against_scipy(dist, params, tr, ref):
    """What the reference's own check_logp does (pymc/testing.py:311-418): density == scipy.stats composition; here plus
    the Jacobian of the default transform (continuous.py:156-163) and central differences for the gradient."""
    from oracle import ir_numpy

    bounds = None
    if tr == "interval":
        bounds = (params[0], params[1])
    elif tr == "interval01":
        tr, bounds = "interval", (0.0, 1.0)
    m = ir.ModelIR(vars=[ir.Var("x", "x", 4, tr, bounds)], priors=[ir.Prior(dist, "x", params)])
    f = ir_numpy.make_logp(m)
    q = np.random.default_rng(1).uniform(-1.2, 1.2, 4)
    lp, g = f(q)
    x = m.constrain(q)["x"]
    if tr == "log":
        jac = q.sum()
    elif tr == "interval":
        lo, hi = bounds
        s = 1 / (1 + np.exp(-q))
        jac = np.sum(np.log(hi - lo) + np.log(s) + np.log1p(-s))
    else:
        jac = 0.0
    assert abs(lp - (np.sum(ref(x)) + jac)) <= 1e-12 * max(1.0, abs(lp))
    assert np.max(np.abs(fd_grad(f, q) - g)) <= 2e-6 * max(1.0, np.max(np.abs(g)))


def test_hierarchical_parameters_and_likelihood_families_by_central_differences():
    from oracle import ir_numpy

    rng = np.random.default_rng(3)
    N, G = 40, 5
    g = rng.integers(0, G, N).astype(np.int32)
    xcov = rng.standard_normal(N)
    vars_ = [ir.Var("m", "m", 1), ir.Var("s_log__", "s", 1, "log"), ir.Var("a", "a", G), ir.Var("b", "b", 1),
             ir.Var("nu_s_log__", "nu_s", 1, "log")]
    pri = [ir.Prior("normal", "m", (0.0, 2.0)), ir.Prior("halfnormal", "s_log__", (1.0,)),
           ir.Prior("normal", "a", (ir.Ref("m"), ir.Ref("s_log__"))), ir.Prior("cauchy", "b", (0.0, ir.Ref("s_log__"))),
           ir.Prior("lognormal", "nu_s_log__", (ir.Ref("m"), 0.5))]
    terms = [ir.Term([("a", g)]), ir.Term([("b", None)], coef=xcov), ir.Term([("s_log__", None), ("a", g), ("b", None)], coef=0.1)]
    for dist, y, kw in [("normal", rng.standard_normal(N), dict(sigma=ir.Ref("nu_s_log__"))),
                        ("studentt", rng.standard_normal(N), dict(sigma=ir.Ref("nu_s_log__"), nu=5.0)),
                        ("bernoulli_logit", (rng.random(N) < 0.4).astype(float), {}),
                        ("poisson_log", rng.poisson(2.0, N).astype(float), {}),
                        ("normal", rng.standard_normal(N), dict(sigma=np.exp(rng.uniform(-0.5, 0.5, N)))),
                        ("normal", rng.standard_normal(N), dict(sigma=0.8))]:
        m = ir.ModelIR(vars=vars_, priors=pri, likelihoods=[ir.Likelihood(dist, y, terms, **kw)])
        f = ir_numpy.make_logp(m)
        q = rng.uniform(-0.8, 0.8, m.n)
        lp, gr = f(q)
        assert np.isfinite(lp)
        assert np.max(np.abs(fd_grad(f, q) - gr)) <= 5e-6 * max(1.0, np.max(np.abs(gr))), dist


def test_specialise_routes_recognised_shapes_to_the_hand_written_kernels():
    es = ir.specialise(ir.eight_schools_ir())
    assert es is not None and es.name == "eight_schools" and es.n == 10
    rd = ir.specialise(ir.radon_ir(n_obs=40, n_counties=7, seed=5))
    ref = models.radon(40, 7, 5)
    assert rd is not None and rd.name == "radon" and rd.n == ref.n
    assert all(np.array_equal(rd.data[k], ref.data[k]) for k in ref.data) and rd.meta["n_counties"] == 7
    assert np.array_equal(rd.initial_point(), ref.initial_point())
    # a different prior scale is NOT the benchmark model: generic path
    other = ir.radon_ir()
    other.priors[0] = ir.Prior("normal", "mu_a", (0.0, 10.0))
    assert ir.specialise(other) is None
    assert ir.specialise(ir.stochvol_ir(T=50)) is None and ir.specialise(ir.varying_intercept_logistic_ir()) is None


def test_extended_specialisation_routes_configs_3_and_4_to_their_hand_kernels():
    """specialise(extended=True): the AR(1) stochastic-volatility IR -> the StochVol kernel's ModelSpec, a Bernoulli-logit GLM with
    beta ~ Normal(0, 1) -> the fused design-matrix kernels' ModelSpec; the specialised spec has the IR's density and gradient
    (NumPy restatements of both), anything that deviates stays on the generic function."""
    from oracle import ir_numpy, logp_numpy

    m = ir.stochvol_ir(T=50)
    sv = ir.specialise(m, extended=True)
    ref = models.stochvol(T=50)
    assert sv is not None and sv.name == "stochvol" and sv.n == ref.n and np.array_equal(sv.data["y"], ref.data["y"])
    assert np.array_equal(sv.initial_point(), ref.initial_point()) and [v.name for v in sv.vars] == [v.name for v in ref.vars]
    f_ir, f_spec = ir_numpy.make_logp(m), logp_numpy.make_logp(sv)
    rng = np.random.default_rng(0)
    for _ in range(3):
        q = m.initial_point() + rng.uniform(-0.5, 0.5, m.n)
        (a, ga), (b, gb) = f_ir(q), f_spec(q)
        assert abs(a - b) <= 1e-11 * abs(b) and np.max(np.abs(ga - gb)) <= 1e-10 * np.max(np.abs(gb))
    off = ir.stochvol_ir(T=50)
    off.ar1[0] = ir.AR1("h", ir.Ref("phi_interval__"), ir.Ref("sigma_log__"), 2.0)  # another init_dist: not the kernel's model
    assert ir.specialise(off, extended=True) is None
    # logistic GLM written as K coefficient columns (what from_pymc produces for dot(X, beta))
    lg = models.logistic(n_rows=300, n_features=5, seed=2)
    X, y = lg.data["X"], lg.data["y"].astype(np.float64)
    terms = [ir.Term([("beta", np.full(300, k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(5)]
    g = ir.ModelIR(vars=[ir.Var("beta", "beta", 5)], priors=[ir.Prior("normal", "beta", (0.0, 1.0))],
                   likelihoods=[ir.Likelihood("bernoulli_logit", y, terms)])
    g.validate()
    assert ir.specialise(g) is None
    sp = ir.specialise(g, extended=True)
    assert sp is not None and sp.name == "logistic" and sp.n == 5 and np.array_equal(sp.data["X"], X)
    assert sp.data["y"].dtype == np.uint8 and np.array_equal(sp.data["y"], lg.data["y"])
    f_ir, f_spec = ir_numpy.make_logp(g), logp_numpy.make_logp(sp)
    for _ in range(3):
        q = rng.uniform(-1, 1, 5)
        (a, ga), (b, gb) = f_ir(q), f_spec(q)
        assert abs(a - b) <= 1e-11 * abs(b) and np.max(np.abs(ga - gb)) <= 1e-10 * np.max(np.abs(gb))
    g.priors[0] = ir.Prior("normal", "beta", (0.0, 2.5))
    assert ir.specialise(g, extended=True) is None


def test_validation_rejects_what_is_outside_the_closed_set():
    v = [ir.Var("x", "x", 3)]
    with pytest.raises(ValueError):
        ir.ModelIR(vars=v, priors=[ir.Prior("weibull", "x", (1.0, 2.0))]).validate()
    with pytest.raises(ValueError):
        ir.ModelIR(vars=v, priors=[ir.Prior("normal", "x", (ir.Ref("x"), 1.0))]).validate()  # parameter must be scalar
    with pytest.raises(ValueError):
        ir.ModelIR(vars=v, likelihoods=[ir.Likelihood("normal", np.zeros(5), [ir.Term([("x", None)])], sigma=1.0)]).validate()
    with pytest.raises(ValueError):
        ir.ModelIR(vars=v, likelihoods=[ir.Likelihood("normal", np.zeros(5), [ir.Term([("x", np.array([0, 1, 2, 3, 0]))])],
                                                      sigma=1.0)]).validate()
    with pytest.raises(ValueError):
        ir.ModelIR(vars=[ir.Var("p", "p", 1, "interval")]).validate()


def test_lowering_fills_the_c_abi_tables():
    m = ir.radon_ir(n_obs=40, n_counties=7, seed=5)
    low = ir.lower(m)
    assert low.n == 19 and [tuple(r) for r in low.vars[:2]] == [(0, 1, 0), (1, 1, 1)]
    c_ir, keep = _lib.build_ir(low)
    assert (c_ir.n_vars, c_ir.n_priors, c_ir.n_liks, c_ir.n_ar1) == (7, 7, 1, 0)
    lik = ctypes.cast(c_ir.liks, ctypes.POINTER(_lib.IrLik))[0]
    assert lik.N == 40 and lik.n_terms == 4 and lik.sigma_kind == ir.SIGMA_REF and lik.sigma.ref == 18
    terms = ctypes.cast(lik.terms, ctypes.POINTER(_lib.IrTerm))
    assert terms[1].n_factors == 2 and terms[1].f[1].offset == 4 and terms[1].f[1].size == 7 and terms[1].f[1].idx
    assert terms[0].coef is None and terms[2].coef


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
IR_MODELS = {
    "eight_schools": ir.eight_schools_ir,
    "radon": ir.radon_ir,
    "radon_small": lambda: ir.radon_ir(40, 7, 5),
    "stochvol_small": lambda: ir.stochvol_ir(T=100, seed=4),   # n = 103: chain = warp
    "stochvol": ir.stochvol_ir,                                 # n = 3003: chain = CTA of 8 warps
    "varying_intercept_logistic": ir.varying_intercept_logistic_ir,
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(IR_MODELS))
def test_ir_device_function_matches_ir_oracle(name):
    from oracle import ir_numpy
    from pymc_b200 import engine

    m = IR_MODELS[name]()
    cm = engine.CompiledModel(m, specialise=False)
    assert cm.spec.name == "ir"
    f = ir_numpy.make_logp(m)
    rng = np.random.default_rng(0)
    nq = 67 if m.n < 1000 else 9
    Q = m.initial_point() + rng.uniform(-1.0, 1.0, (nq, m.n))
    lp, g = cm.logp_dlogp(Q)
    lo = np.array([f(q)[0] for q in Q])
    go = np.array([f(q)[1] for q in Q])
    assert np.max(np.abs(lp - lo) / np.abs(lo)) <= 1e-12
    assert np.max(np.abs(g - go) / np.max(np.abs(go), axis=1, keepdims=True)) <= 1e-12
    lp2, g2 = cm.logp_dlogp(Q)  # deterministic: no atomics anywhere in the gradient
    assert np.array_equal(lp, lp2) and np.array_equal(g, g2)


@pytest.mark.gpu
@pytest.mark.parametrize("name,builder", [("eight_schools_fixed", ir.eight_schools_ir), ("radon_fixed", ir.radon_ir),
                                          ("stochvol_small_fixed", lambda: ir.stochvol_ir(T=100, seed=4))])
def test_ir_models_reproduce_the_reference_goldens_without_model_specific_cuda(golden, name, builder):
    """VERDICT r1 next #8: Eight Schools and Radon expressed purely in IR reproduce today's goldens (identical tree
    statistics for every draw, positions to 1e-9) on the GENERIC device function."""
    from b200_helpers import discrete_equal, gpu_free_run
    from pymc_b200 import engine

    d = golden(name)
    cm = engine.CompiledModel(builder(), specialise=False)
    res, _ = gpu_free_run(cm, d, name)
    for c in range(len(d["seeds"])):
        st = {k: v[c] for k, v in res.stats.items()}
        assert discrete_equal(st, d, c).all(), (name, c)
        assert np.max(np.abs(res.draws[c] - d["draws_q"][c])) <= 1e-9


@pytest.mark.gpu
def test_new_model_runs_with_no_new_cuda_and_matches_the_oracle_sampler():
    """A model no kernel was written for (centred varying-intercept logistic regression): fixed-step NUTS on the device
    equals the oracle NUTS on the IR's NumPy logp draw by draw; an adaptive run recovers the oracle's posterior."""
    from oracle import ir_numpy

    m = ir.varying_intercept_logistic_ir()
    f = ir_numpy.make_logp(m)
    fixed_step_against_oracle(m, f, 0.05, specialise=True, q0_seed=5)
    adaptive_against_oracle(m, f, specialise=True, chain_seed=21, spread=1, philox_seed=3, oracle_seed=100, se_bound=5.0,
                            max_divergence=0.02)


@pytest.mark.gpu
def test_pointwise_log_likelihood_matches_oracle_and_sums_to_the_likelihood_term():
    """pm.compute_log_likelihood's group (pymc/stats/log_density.py:31-77) from the device: log p(y_i | draw) per draw."""
    from scipy import stats as st

    from pymc_b200 import engine

    m = ir.radon_ir(60, 5, 3)
    cm = engine.CompiledModel(m, specialise=False)
    rng = np.random.default_rng(4)
    q = m.initial_point() + rng.uniform(-0.5, 0.5, (3, 7, m.n))
    ll = cm.pointwise_loglik(q)
    assert ll.shape == (3, 7, 60)
    c = m.constrain(q)
    L = m.likelihoods[0]
    county, floor = L.terms[1].factors[1][1], L.terms[2].coef
    mu = (c["mu_a"][..., None] + c["sigma_a"][..., None] * c["a"][..., county]
          + (c["mu_b"][..., None] + c["sigma_b"][..., None] * c["b"][..., county]) * floor)
    want = st.norm(mu, c["eps"][..., None]).logpdf(L.y)
    np.testing.assert_allclose(ll, want, rtol=1e-12, atol=1e-12)
    m2 = ir.varying_intercept_logistic_ir()
    cm2 = engine.CompiledModel(m2)
    q2 = rng.uniform(-1, 1, (5, m2.n))
    ll2 = cm2.pointwise_loglik(q2)
    c2 = m2.constrain(q2)
    L2 = m2.likelihoods[0]
    eta = c2["alpha"][:, L2.terms[0].factors[0][1]] + sum(c2["beta"][:, [k]] * L2.terms[1 + k].coef for k in range(3))
    want2 = L2.y * eta - np.logaddexp(0.0, eta)
    np.testing.assert_allclose(ll2, want2, rtol=1e-12, atol=1e-13)
