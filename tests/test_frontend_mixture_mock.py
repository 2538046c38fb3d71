"""CPU: ``from_pymc`` on imitation graphs (tests/test_frontend_mock.py's stand-ins) of finite mixtures.

pm.NormalMixture("y", w, mu, sigma) and pm.Mixture("y", w, pm.Poisson.dist(lam, shape=K)) build a Mixture of ONE batched
component whose parameters PyMC resizes to (N, K) through DimShuffle / broadcast layers (pymc/distributions/mixture.py:
469-494, :529-546); w is a free pm.Dirichlet (SimplexTransform) or a constant K-vector.  Each spelling must lower to an IR
with the density of the hand-built IR; tau=, other component families, other weight forms, per-observation parameters, a
Dirichlet variable used elsewhere and list-form mixtures are refused by name."""
import numpy as np
import pytest
from test_frontend_mock import Constant, FakeModel, LogTransform, SharedVariable, apply, bcast, elem, fake_pytensor, rv  # noqa: F401
from test_frontend_mock import Dot, same_density

from pymc_b200 import ir

K, N = 3, 40


class SimplexTransform:
    pass


def ordered(positive=False):
    return type("Ordered", (), {"positive": positive, "ascending": True})()


def oracle(m):
    from oracle import ir_numpy_mixture

    return ir_numpy_mixture.make_logp(m)


def _data(dist, seed=5):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, 2))
    y = rng.normal(0.0, 2.0, N) if dist == "normal" else rng.poisson(3.0, N).astype(np.float64)
    return X, y


def _weights(M, kind, vars_, priors):
    if kind == "dirichlet":
        w = M.free(rv("DirichletRV", "w", Constant(np.ones(K))), K - 1, SimplexTransform(), suffix="_simplex__")
        vars_.append(ir.Var("w_simplex__", "w", K - 1, "simplex"))
        priors.append(ir.Prior("dirichlet", "w_simplex__", (np.ones(K),)))
        return bcast(w), ir.Ref("w_simplex__")
    c = np.array([0.2, 0.3, 0.5])
    return Constant(np.broadcast_to(c, (N, K)).copy()), c


def _eta(M, X, vars_, priors):
    beta = M.free(rv("NormalRV", "beta", Constant(0.0), Constant(1.0)), 2)
    vars_.append(ir.Var("beta", "beta", 2))
    priors.append(ir.Prior("normal", "beta", (0.0, 1.0)))
    return apply(Dot(), SharedVariable(X), beta), [ir.Term([("beta", None)], coef=X)]


def normal_model(weights="dirichlet", mu="ordered", sigma="vector", eta=None):
    """pm.NormalMixture("y", w, mu, sigma): mu a free ordered K-vector or constants, optionally eta[:, None] + mu (or
    mu + eta[:, None]); sigma a K-vector or scalar free RV, or one or K constants."""
    X, y = _data("normal")
    M, vars_, priors = FakeModel("nm"), [], []
    w, w_ir = _weights(M, weights, vars_, priors)
    if mu == "ordered":
        m = M.free(rv("NormalRV", "mu", Constant(0.0), Constant(10.0)), K, ordered(), suffix="_ordered__")
        vars_.append(ir.Var("mu_ordered__", "mu", K, "ordered"))
        priors.append(ir.Prior("normal", "mu_ordered__", (0.0, 10.0)))
        loc, mu_ir = bcast(m), ir.Ref("mu_ordered__")
    else:
        loc, mu_ir = Constant(np.array([-2.0, 0.0, 2.0])), np.array([-2.0, 0.0, 2.0])
    if sigma in ("vector", "scalar"):
        s = M.free(rv("HalfNormalRV", "sigma", Constant(0.0), Constant(2.0)), K if sigma == "vector" else 1, LogTransform())
        vars_.append(ir.Var("sigma_log__", "sigma", K if sigma == "vector" else 1, "log"))
        priors.append(ir.Prior("halfnormal", "sigma_log__", (2.0,)))
        sg, s_ir = bcast(s), ir.Ref("sigma_log__")
    elif sigma == "const":
        sg, s_ir = Constant(1.5), 1.5
    else:
        sg, s_ir = Constant(np.array([0.5, 1.0, 2.0])), np.array([0.5, 1.0, 2.0])
    terms = []
    if eta is not None:
        e, terms = _eta(M, X, vars_, priors)
        loc = elem("Add", bcast(e), loc) if eta == "first" else elem("Add", loc, bcast(e))
    M.observe(rv("MixtureRV", "y", w, rv("NormalRV", None, bcast(loc), bcast(sg))), y)
    ref = ir.ModelIR(vars=vars_, priors=priors,
                     likelihoods=[ir.Likelihood("normal_mixture", y, terms, sigma=s_ir, weights=w_ir, components=mu_ir)])
    return M, ref


def poisson_model(weights="dirichlet", lam="ordered_positive", eta=None):
    """pm.Mixture("y", w, pm.Poisson.dist(lam, shape=K)): lam a free ordered_positive K-vector or constants, optionally
    pm.math.exp(eta)[:, None] * lam."""
    X, y = _data("poisson")
    M, vars_, priors = FakeModel("pm"), [], []
    w, w_ir = _weights(M, weights, vars_, priors)
    if lam == "ordered_positive":
        lv = M.free(rv("NormalRV", "lam", Constant(0.0), Constant(20.0)), K, ordered(True), suffix="_ordered__")
        vars_.append(ir.Var("lam_ordered__", "lam", K, "ordered_positive"))
        priors.append(ir.Prior("normal", "lam_ordered__", (0.0, 20.0)))
        rate, lam_ir = bcast(lv), ir.Ref("lam_ordered__")
    else:
        rate, lam_ir = Constant(np.array([0.5, 3.0, 9.0])), np.array([0.5, 3.0, 9.0])
    terms = []
    if eta is not None:
        e, terms = _eta(M, X, vars_, priors)
        rate = elem("Mul", bcast(elem("Exp", e)), rate)
    M.observe(rv("MixtureRV", "y", w, rv("PoissonRV", None, bcast(rate))), y)
    ref = ir.ModelIR(vars=vars_, priors=priors,
                     likelihoods=[ir.Likelihood("poisson_mixture", y, terms, weights=w_ir, components=lam_ir)])
    return M, ref


SPELLINGS = {
    "normal_dirichlet_ordered_vector_sigma": lambda: normal_model(),
    "normal_dirichlet_scalar_sigma_eta_first": lambda: normal_model(sigma="scalar", eta="first"),
    "normal_dirichlet_const_sigma_eta_last": lambda: normal_model(sigma="const", eta="last"),
    "normal_const_weights_const_mu_const_sigmas": lambda: normal_model("const", "const", "consts", eta="first"),
    "poisson_dirichlet_ordered_positive": lambda: poisson_model(),
    "poisson_dirichlet_exp_eta": lambda: poisson_model(eta=True),
    "poisson_const_weights_const_lam_exp_eta": lambda: poisson_model("const", "const", eta=True),
}


@pytest.mark.parametrize("name", list(SPELLINGS))
def test_each_spelling_lowers_to_the_hand_built_density(fake_pytensor, name):
    from pymc_b200 import from_pymc

    M, ref = SPELLINGS[name]()
    m = from_pymc(M)
    L, R = m.likelihoods[0], ref.likelihoods[0]
    assert L.dist == R.dist and type(L.weights) is type(R.weights) and type(L.components) is type(R.components)
    assert bool(L.terms) == bool(R.terms)
    same_density(oracle(m), oracle(ref), m, ref, spread=0.5)
    low = ir.lower(ir.fuse_design_columns(m))
    assert low.liks[0]["nu"] == float(K) and len(low.liks[0]["mix"]) == (3 if R.dist == "normal_mixture" else 2)
    if isinstance(R.weights, ir.Ref):
        assert low.priors[0][0] == ir.PRIOR_DISTS["dirichlet"][0] and tuple(low.vars[0]) == (0, K - 1, 5)


def _refused(build, match):
    from pymc_b200 import from_pymc

    with pytest.raises(NotImplementedError, match=match):
        from_pymc(build())


def _base():
    X, y = _data("normal")
    M = FakeModel("bad")
    w = M.free(rv("DirichletRV", "w", Constant(np.ones(K))), K - 1, SimplexTransform(), suffix="_simplex__")
    mu = M.free(rv("NormalRV", "mu", Constant(0.0), Constant(10.0)), K, ordered(), suffix="_ordered__")
    return M, w, mu, y


def test_other_forms_are_refused_by_name(fake_pytensor):
    def tau():
        M, w, mu, y = _base()
        t = M.free(rv("GammaRV", "tau", Constant(2.0), Constant(1.0)), K, LogTransform())
        M.observe(rv("MixtureRV", "y", bcast(w), rv("NormalRV", None, bcast(mu), bcast(elem("Pow", t, Constant(-0.5))))), y)
        return M

    def gamma_components():
        M, w, mu, y = _base()
        M.observe(rv("MixtureRV", "y", bcast(w), rv("GammaRV", None, Constant(2.0), bcast(mu))), np.abs(y))
        return M

    def normal_weights():
        M, w, mu, y = _base()
        v = M.free(rv("NormalRV", "v", Constant(0.0), Constant(1.0)), K)
        M.observe(rv("MixtureRV", "y", bcast(v), rv("NormalRV", None, bcast(mu), Constant(1.0))), y)
        return M

    def softmax_weights():
        M, w, mu, y = _base()
        M.observe(rv("MixtureRV", "y", elem("Softmax", bcast(mu)), rv("NormalRV", None, bcast(mu), Constant(1.0))), y)
        return M

    def per_obs_weights():
        M, w, mu, y = _base()
        c = np.random.default_rng(0).dirichlet(np.ones(K), N)
        M.observe(rv("MixtureRV", "y", Constant(c), rv("NormalRV", None, bcast(mu), Constant(1.0))), y)
        return M

    def per_obs_mu():
        M, w, mu, y = _base()
        big = M.free(rv("NormalRV", "m2", Constant(0.0), Constant(1.0)), N * K)
        M.observe(rv("MixtureRV", "y", bcast(w), rv("NormalRV", None, big, Constant(1.0))), y)
        return M

    def per_obs_sigma():
        M, w, mu, y = _base()
        s = np.random.default_rng(0).uniform(0.5, 2.0, (N, K))
        M.observe(rv("MixtureRV", "y", bcast(w), rv("NormalRV", None, bcast(mu), Constant(s))), y)
        return M

    def simplex_as_mu():
        M, w, mu, y = _base()
        M.observe(rv("MixtureRV", "y", bcast(w), rv("NormalRV", None, bcast(w), Constant(1.0))), y)
        return M

    def simplex_in_a_predictor():
        M, w, mu, y = _base()
        M.observe(rv("MixtureRV", "y", bcast(w), rv("NormalRV", None, bcast(mu), Constant(1.0))), y)
        M.observe(rv("NormalRV", "z", elem("Mul", Constant(2.0), w), Constant(1.0)), y[:K - 1])
        return M

    def random_a():
        M = FakeModel("bad")
        a = M.free(rv("HalfNormalRV", "a", Constant(0.0), Constant(1.0)), 1, LogTransform())
        M.free(rv("DirichletRV", "w", bcast(a)), K - 1, SimplexTransform(), suffix="_simplex__")
        return M

    def list_form():
        M, w, mu, y = _base()
        M.observe(rv("MixtureRV", "y", bcast(w), rv("NormalRV", None, Constant(0.0), Constant(1.0)),
                     rv("NormalRV", None, Constant(2.0), Constant(1.0))), y)
        return M

    _refused(tau, r"NormalMixture\(tau=\.\.\.\)")
    _refused(gamma_components, "a mixture of GammaRV components is outside the closed set")
    _refused(normal_weights, "the weights of a mixture are a free pm.Dirichlet or a constant K-vector")
    _refused(softmax_weights, "the weights of a mixture are a free pm.Dirichlet or a constant K-vector")
    _refused(per_obs_weights, "per-observation weights")
    _refused(per_obs_mu, "per-observation mu")
    _refused(per_obs_sigma, "per-observation sigma")
    _refused(simplex_as_mu, "w: " + ir.SIMPLEX_USE)
    _refused(simplex_in_a_predictor, "w: " + ir.SIMPLEX_USE)
    _refused(random_a, "a pm.Dirichlet with a random a")
    _refused(list_form, "a list-of-components pm.Mixture / pm.NormalMixture is outside the closed set")


def test_a_one_component_mixture_is_refused_by_the_support_rule(fake_pytensor):
    from pymc_b200 import from_pymc

    X, y = _data("normal")
    M = FakeModel("k1")
    M.observe(rv("MixtureRV", "y", Constant(np.ones((N, 1))), rv("NormalRV", None, Constant(np.zeros(1)), Constant(1.0))), y)
    with pytest.raises(ValueError, match="write the plain likelihood"):
        from_pymc(M)
