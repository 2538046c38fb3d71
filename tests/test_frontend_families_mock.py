"""CPU: ``from_pymc`` on imitation graphs (tests/test_frontend_mock.py's stand-ins) of the count and positive likelihoods --
Binomial with logit_p / p = sigmoid(eta), NegativeBinomial(mu = exp(eta), alpha) as PyMC stores it, (n = alpha,
p = alpha / (mu + alpha)), and Gamma(alpha, beta = alpha / exp(eta) or alpha * exp(-eta)) as (alpha, scale = 1 / beta).
Each graph must lower to an IR with the density of the hand-built IR; other spellings are refused by name."""
import numpy as np
import pytest

from test_frontend_mock import Constant, DimShuffle, FakeModel, LogTransform, apply, bcast, elem, fake_pytensor, rv  # noqa: F401
from test_frontend_mock import same_density

from oracle.ir_numpy_families import make_logp
from pymc_b200 import ir


def _regression(M, rng, N):
    """b0 + b1 * x as a graph, and the same predictor as IR terms."""
    x = rng.standard_normal(N)
    b0 = M.free(rv("NormalRV", "b0", Constant(0.0), Constant(2.0)), 1)
    b1 = M.free(rv("NormalRV", "b1", Constant(0.0), Constant(1.0)), 1)
    eta = elem("Add", bcast(b0), elem("Mul", bcast(b1), Constant(x)))
    vars_ = [ir.Var("b0", "b0", 1), ir.Var("b1", "b1", 1)]
    priors = [ir.Prior("normal", "b0", (0.0, 2.0)), ir.Prior("normal", "b1", (0.0, 1.0))]
    return eta, vars_, priors, [ir.Term([("b0", None)]), ir.Term([("b1", None)], coef=x)]


@pytest.mark.parametrize("spelling", ["logit_p", "p_sigmoid", "scalar_trials"])
def test_binomial_graphs_lower_to_the_binomial_logit_likelihood(fake_pytensor, spelling):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(1)
    N = 30
    M = FakeModel("binomial")
    eta, vars_, priors, terms = _regression(M, rng, N)
    trials = np.full(N, 12.0) if spelling == "scalar_trials" else rng.integers(1, 20, N).astype(float)
    y = np.floor(trials * rng.random(N))
    p = elem("Sigmoid", eta) if spelling != "p_sigmoid" else bcast(elem("Sigmoid", eta))
    M.observe(rv("BinomialRV", "y", Constant(12.0 if spelling == "scalar_trials" else trials), p), y)
    m = from_pymc(M)
    L = m.likelihoods[0]
    assert L.dist == "binomial_logit" and (L.trials == 12.0 if spelling == "scalar_trials" else np.array_equal(L.trials, trials))
    ref = ir.ModelIR(vars=vars_, priors=priors, likelihoods=[ir.Likelihood("binomial_logit", y, terms,
                                                                           trials=12.0 if spelling == "scalar_trials" else trials)])
    same_density(make_logp(m), make_logp(ref), m, ref, spread=0.7)


@pytest.mark.parametrize("alpha_kind,add_order,op_name", [("ref", "mu_first", "NegBinomialRV"), ("ref", "alpha_first", "NBinomRV"),
                                                          ("const", "mu_first", "NegBinomialRV")])
def test_negative_binomial_graph_lowers_with_a_random_or_constant_alpha(fake_pytensor, alpha_kind, add_order, op_name):
    """pm.NegativeBinomial(mu=exp(eta), alpha=a) holds (n = a, p = a / (exp(eta) + a)) (discrete.py:700-723)."""
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(2)
    N = 40
    M = FakeModel("negbin")
    eta, vars_, priors, terms = _regression(M, rng, N)
    y = rng.poisson(3.0, N).astype(float)
    if alpha_kind == "ref":
        a = M.free(rv("ExponentialRV", "alpha", Constant(1.0)), 1, LogTransform())
        vars_.append(ir.Var("alpha_log__", "alpha", 1, "log"))
        priors.append(ir.Prior("exponential", "alpha_log__", (1.0,)))
        alpha = ir.Ref("alpha_log__")
    else:
        a = Constant(2.5)
        alpha = 2.5
    mu = elem("Exp", eta)
    den = elem("Add", mu, bcast(a)) if add_order == "mu_first" else elem("Add", bcast(a), mu)
    M.observe(rv(op_name, "y", a, elem("TrueDiv", bcast(a), den)), y)
    m = from_pymc(M)
    assert m.likelihoods[0].dist == "negative_binomial_log" and m.likelihoods[0].alpha == alpha
    ref = ir.ModelIR(vars=vars_, priors=priors, likelihoods=[ir.Likelihood("negative_binomial_log", y, terms, alpha=alpha)])
    same_density(make_logp(m), make_logp(ref), m, ref, spread=0.7, seed=1)


@pytest.mark.parametrize("beta_form", ["a_over_exp", "a_times_exp_neg", "exp_neg_times_a"])
def test_gamma_graph_lowers_with_a_random_shape(fake_pytensor, beta_form):
    """pm.Gamma(alpha=a, beta=...) holds (alpha, scale = reciprocal(beta)) (continuous.py:2478-2510)."""
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(3)
    N = 35
    M = FakeModel("gamma")
    eta, vars_, priors, terms = _regression(M, rng, N)
    y = rng.gamma(2.0, 1.5, N)
    a = M.free(rv("HalfNormalRV", "alpha", Constant(0.0), Constant(2.0)), 1, LogTransform())
    vars_.append(ir.Var("alpha_log__", "alpha", 1, "log"))
    priors.append(ir.Prior("halfnormal", "alpha_log__", (2.0,)))
    if beta_form == "a_over_exp":
        beta = elem("TrueDiv", bcast(a), elem("Exp", eta))
    elif beta_form == "a_times_exp_neg":
        beta = elem("Mul", bcast(a), elem("Exp", elem("Neg", eta)))
    else:
        beta = elem("Mul", elem("Exp", elem("Neg", eta)), bcast(a))
    M.observe(rv("GammaRV", "y", a, elem("Reciprocal", beta)), y)
    m = from_pymc(M)
    assert m.likelihoods[0].dist == "gamma_log" and m.likelihoods[0].alpha == ir.Ref("alpha_log__")
    ref = ir.ModelIR(vars=vars_, priors=priors, likelihoods=[ir.Likelihood("gamma_log", y, terms, alpha=ir.Ref("alpha_log__"))])
    same_density(make_logp(m), make_logp(ref), m, ref, spread=0.7, seed=2)


def test_other_spellings_of_the_families_are_refused_by_name(fake_pytensor):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(4)
    N = 10
    y = rng.poisson(2.0, N).astype(float)

    def model(obs):
        M = FakeModel()
        eta, *_ = _regression(M, rng, N)
        a = M.free(rv("ExponentialRV", "alpha", Constant(1.0)), 1, LogTransform())
        M.observe(obs(eta, a), y)
        return M

    cases = [
        ("Binomial", lambda eta, a: rv("BinomialRV", "y", Constant(10.0), elem("Tanh", eta))),              # p not sigmoid(eta)
        ("Binomial", lambda eta, a: rv("BinomialRV", "y", bcast(a), elem("Sigmoid", eta))),                 # random trials
        ("NegativeBinomial", lambda eta, a: rv("NegBinomialRV", "y", a, elem("Sigmoid", eta))),             # p given directly
        ("NegativeBinomial", lambda eta, a: rv("NegBinomialRV", "y", a,
                                               elem("TrueDiv", Constant(3.0), elem("Add", elem("Exp", eta), bcast(a))))),  # alpha mismatch
        ("NegativeBinomial", lambda eta, a: rv("NegBinomialRV", "y", a,
                                               elem("TrueDiv", bcast(a), elem("Add", eta, bcast(a))))),     # mu not exp(eta)
        ("Gamma", lambda eta, a: rv("GammaRV", "y", a, elem("Exp", eta))),                                  # scale = exp(eta)
        ("Gamma", lambda eta, a: rv("GammaRV", "y", a, elem("Reciprocal", elem("Mul", Constant(2.0), elem("Exp", elem("Neg", eta)))))),
        ("Gamma", lambda eta, a: rv("GammaRV", "y", a, elem("Reciprocal", elem("TrueDiv", bcast(a), eta)))),
    ]
    for what, obs in cases:
        with pytest.raises(NotImplementedError, match=f"pm.{what}"):
            from_pymc(model(obs))
