"""CPU: ``from_pymc`` on imitation graphs (tests/test_frontend_mock.py's stand-ins) of censored and truncated Normal
observations: pm.Censored(pm.Normal.dist(eta, sigma), lower, upper) as a CensoredRV with dist params (base, lower, upper),
and pm.TruncatedNormal(eta, sigma, lower, upper) -- also what pm.Truncated(pm.Normal.dist(...)) becomes.  Each graph must
lower to an IR with the density of the hand-built IR.  Other bases, including a TruncatedRV (the base RV's inputs, then
lower and upper, its op in ``base_rv_op``), and random bounds are refused by name."""
import numpy as np
import pytest
from test_frontend_mock import Constant, FakeModel, LogTransform, Variable, apply, bcast, elem, fake_pytensor, rv  # noqa: F401
from test_frontend_mock import same_density

from oracle.ir_numpy_bounded import make_logp
from pymc_b200 import ir


def _model(rng, N, obs):
    """b0 + b1 x and sigma ~ HalfNormal(1) as a graph; obs(M, eta, sigma) adds the observed RV."""
    x = rng.standard_normal(N)
    M = FakeModel("bounded")
    b0 = M.free(rv("NormalRV", "b0", Constant(0.0), Constant(2.0)), 1)
    b1 = M.free(rv("NormalRV", "b1", Constant(0.0), Constant(1.0)), 1)
    s = M.free(rv("HalfNormalRV", "sigma", Constant(0.0), Constant(1.0)), 1, LogTransform())
    eta = elem("Add", bcast(b0), elem("Mul", bcast(b1), Constant(x)))
    obs(M, eta, s)
    vars_ = [ir.Var("b0", "b0", 1), ir.Var("b1", "b1", 1), ir.Var("sigma_log__", "sigma", 1, "log")]
    priors = [ir.Prior("normal", "b0", (0.0, 2.0)), ir.Prior("normal", "b1", (0.0, 1.0)), ir.Prior("halfnormal", "sigma_log__", (1.0,))]
    return M, vars_, priors, [ir.Term([("b0", None)]), ir.Term([("b1", None)], coef=x)]


BOUND_FORMS = {  # (lower, upper) as the graph holds them -> as the IR holds them
    "scalar": ((-0.5, 1.0), (-0.5, 1.0)),
    "array": ((np.linspace(-1.5, -0.5, 30), np.linspace(0.8, 2.0, 30)), None),
    "open_lower": ((-np.inf, 1.0), (None, 1.0)),
    "open_upper": ((-0.5, np.inf), (-0.5, None)),
    "mixed_array": ((np.where(np.arange(30) % 3 == 0, -np.inf, -0.5), np.where(np.arange(30) % 4 == 0, np.inf, 1.0)), None),
}


@pytest.mark.parametrize("form", list(BOUND_FORMS))
@pytest.mark.parametrize("spelling", ["Censored", "TruncatedNormal"])
def test_bounded_graphs_lower_to_the_bounded_likelihoods(fake_pytensor, spelling, form):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(7)
    N = 30
    (lo, hi), want = BOUND_FORMS[form]
    want = want if want is not None else (lo, hi)
    lo_a, hi_a = np.broadcast_to(lo, (N,)), np.broadcast_to(hi, (N,))
    y = np.clip(rng.normal(0.3, 1.0, N), lo_a, hi_a)
    if spelling != "Censored":
        y = np.clip(y, np.nextafter(lo_a, np.inf), np.nextafter(hi_a, -np.inf))

    def obs(M, eta, s):
        if spelling == "TruncatedNormal":
            r = rv("TruncatedNormalRV", "y", eta, bcast(s), Constant(lo), Constant(hi))
        else:
            r = rv("CensoredRV", "y", rv("NormalRV", None, eta, bcast(s)), Constant(lo), Constant(hi))
        M.observe(r, y)

    M, vars_, priors, terms = _model(rng, N, obs)
    m = from_pymc(M)
    L = m.likelihoods[0]
    dist = "censored_normal" if spelling == "Censored" else "truncated_normal"
    assert L.dist == dist and L.sigma == ir.Ref("sigma_log__")
    for got, exp in zip((L.lower, L.upper), want):
        assert (got is None and exp is None) or np.array_equal(got, exp), (got, exp)
    ref = ir.ModelIR(vars=vars_, priors=priors, likelihoods=[ir.Likelihood(dist, y, terms, sigma=ir.Ref("sigma_log__"),
                                                                           lower=want[0], upper=want[1])])
    same_density(make_logp(m), make_logp(ref), m, ref, spread=0.7)


def truncated_rv(name, base_op, *base_params, lower, upper):
    """A TruncatedRV as PyMC builds it: the base RV's inputs (rng, size, parameters), then lower and upper."""
    op = type("TruncatedRV", (), {"base_rv_op": type(base_op, (), {})(),
                                  "dist_params": lambda self, node: node.inputs[2:]})()
    return apply(op, Variable("rng"), Constant(np.array([])), *base_params, lower, upper, name=name)


def test_other_bases_and_random_bounds_are_refused_by_name(fake_pytensor):
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(8)
    N = 10
    y = np.clip(rng.poisson(2.0, N).astype(float), 0.0, 4.0)

    def model(obs):
        M, *_ = _model(rng, N, obs)
        return M

    cases = [
        ("pm.Censored of StudentTRV", lambda M, eta, s: M.observe(
            rv("CensoredRV", "y", rv("StudentTRV", None, Constant(4.0), eta, bcast(s)), Constant(0.0), Constant(4.0)), y)),
        ("pm.Censored of PoissonRV", lambda M, eta, s: M.observe(
            rv("CensoredRV", "y", rv("PoissonRV", None, elem("Exp", eta)), Constant(0.0), Constant(4.0)), y)),
        ("pm.Truncated of GammaRV", lambda M, eta, s: M.observe(
            truncated_rv("y", "GammaRV", Constant(2.0), elem("Exp", eta), lower=Constant(0.0), upper=Constant(5.0)), y + 0.5)),
        # a Laplace base whose location is a free Normal RV: still named by its base op, not taken for a Normal base
        ("pm.Truncated of LaplaceRV", lambda M, eta, s: M.observe(
            truncated_rv("y", "LaplaceRV", M.free_RVs[0], bcast(s), lower=Constant(-1.0), upper=Constant(5.0)), y)),
        ("random bounds", lambda M, eta, s: M.observe(
            rv("CensoredRV", "y", rv("NormalRV", None, eta, bcast(s)), bcast(s), Constant(np.inf)), y)),
        ("random bounds", lambda M, eta, s: M.observe(rv("TruncatedNormalRV", "y", eta, bcast(s), Constant(-1.0), eta), y)),
    ]
    for what, obs in cases:
        with pytest.raises(NotImplementedError, match=what):
            from_pymc(model(obs))
