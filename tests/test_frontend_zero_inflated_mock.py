"""CPU: ``from_pymc`` on imitation graphs (tests/test_frontend_mock.py's stand-ins) of zero-inflated and hurdle regressions.

pm.ZeroInflatedPoisson / Binomial / NegativeBinomial build a Mixture of [DiracDelta(0), f] with weights
stack([1 - psi, psi], axis=-1) (pymc/distributions/mixture.py:560-574); pm.HurdlePoisson / NegativeBinomial / Gamma a
_Hurdle of [DiracDelta(0), Truncated(f, lower=1)] (Gamma: f itself, :812-844).  Each graph must lower to an IR with the
density of the hand-built IR, for psi a constant, a scalar free RV (logodds transform) and invlogit of a linear predictor;
HurdleLogNormal, other mixtures and other forms of psi are refused by name."""
import numpy as np
import pytest
from test_frontend_bounded_mock import truncated_rv
from test_frontend_mock import Constant, FakeModel, LogTransform, SharedVariable, apply, bcast, elem, fake_pytensor, rv  # noqa: F401
from test_frontend_mock import AdvancedSubtensor1, Dot, Join, same_density
from test_ir_zero_inflated import oracle

from pymc_b200 import ir


class LogOddsTransform:
    pass


def weights(psi):
    """pt.stack([1 - psi, psi], axis=-1)"""
    return apply(Join(), Constant(-1), bcast(elem("Sub", Constant(1.0), psi)), bcast(psi))


def dirac():
    return rv("DiracDeltaRV", None, Constant(0))


def _component(dist, eta, alpha, trials):
    fam = ir.ZI_FAMILY[dist]
    if fam == "poisson_log":
        base = ("PoissonRV", (elem("Exp", eta),))
    elif fam == "binomial_logit":
        base = ("BinomialRV", (Constant(trials), elem("Sigmoid", eta)))
    elif fam == "negative_binomial_log":  # (n = alpha, p = alpha / (mu + alpha))
        base = ("NegBinomialRV", (alpha, elem("TrueDiv", alpha, elem("Add", elem("Exp", eta), alpha))))
    else:  # (alpha, scale = reciprocal(alpha / exp(eta)))
        return rv("GammaRV", None, alpha, elem("Reciprocal", elem("TrueDiv", alpha, elem("Exp", eta))))
    if dist.startswith("hurdle"):
        return truncated_rv(None, base[0], *base[1], lower=Constant(1), upper=Constant(np.inf))
    return rv(base[0], None, *base[1])


def _model(dist, psi_kind, seed=3, N=40):
    rng = np.random.default_rng(seed)
    fam = ir.ZI_FAMILY[dist]
    g = rng.integers(0, 4, N).astype(np.int32)
    X, Z = rng.standard_normal((N, 2)), rng.standard_normal((N, 2))
    trials = rng.integers(0, 9, N).astype(np.float64)
    y = rng.gamma(2.0, 1.0, N) if fam == "gamma_log" else rng.integers(0, 5, N).astype(np.float64)
    if fam == "binomial_logit":
        y = np.minimum(y, trials)
    y[rng.random(N) < 0.3] = 0.0
    M = FakeModel("zi")
    a = M.free(rv("NormalRV", "a", Constant(0.0), Constant(1.0)), 4)
    beta = M.free(rv("NormalRV", "beta", Constant(0.0), Constant(1.0)), 2)
    vars_ = [ir.Var("a", "a", 4), ir.Var("beta", "beta", 2)]
    priors = [ir.Prior("normal", "a", (0.0, 1.0)), ir.Prior("normal", "beta", (0.0, 1.0))]
    alpha, kw = None, {}
    if fam in ir.DISPERSION_LIKS:
        alpha = M.free(rv("HalfNormalRV", "alpha", Constant(0.0), Constant(2.0)), 1, LogTransform())
        vars_.append(ir.Var("alpha_log__", "alpha", 1, "log"))
        priors.append(ir.Prior("halfnormal", "alpha_log__", (2.0,)))
        kw["alpha"] = ir.Ref("alpha_log__")
    if fam == "binomial_logit":
        kw["trials"] = trials
    if psi_kind == "const":
        psi, p_ir = Constant(0.7), 0.7
    elif psi_kind == "var":
        psi = M.free(rv("BetaRV", "psi", Constant(2.0), Constant(2.0)), 1, LogOddsTransform(), suffix="_logodds__")
        vars_.append(ir.Var("psi_logodds__", "psi", 1, "interval", bounds=(0.0, 1.0)))
        priors.append(ir.Prior("beta", "psi_logodds__", (2.0, 2.0)))
        p_ir = ir.Ref("psi_logodds__")
    else:
        g0 = M.free(rv("NormalRV", "g0", Constant(0.0), Constant(1.5)), 1)
        gam = M.free(rv("NormalRV", "gamma", Constant(0.0), Constant(1.0)), 2)
        vars_ += [ir.Var("g0", "g0", 1), ir.Var("gamma", "gamma", 2)]
        priors += [ir.Prior("normal", "g0", (0.0, 1.5)), ir.Prior("normal", "gamma", (0.0, 1.0))]
        psi = elem("Sigmoid", elem("Add", bcast(g0), apply(Dot(), SharedVariable(Z), gam)))
        p_ir = ir.Linear([ir.Term([("g0", None)])] + [ir.Term([("gamma", np.full(N, k, dtype=np.int32))], coef=Z[:, k].copy())
                                                      for k in range(2)])
    eta = elem("Add", apply(AdvancedSubtensor1(), a, Constant(g)), apply(Dot(), SharedVariable(X), beta))
    op = "_HurdleRV" if dist.startswith("hurdle") else "MixtureRV"
    M.observe(rv(op, "y", weights(psi), dirac(), _component(dist, eta, alpha, trials)), y)
    terms = [ir.Term([("a", g)])] + [ir.Term([("beta", np.full(N, k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(2)]
    ref = ir.ModelIR(vars=vars_, priors=priors, likelihoods=[ir.Likelihood(dist, y, terms, psi=p_ir, **kw)])
    return M, ref


@pytest.mark.parametrize("psi_kind", ["const", "var", "logit"])
@pytest.mark.parametrize("dist", ir.ZI_LIKS)
def test_each_spelling_lowers_to_the_hand_built_density(fake_pytensor, dist, psi_kind):
    from pymc_b200 import from_pymc

    M, ref = _model(dist, psi_kind)
    m = from_pymc(M)
    L = m.likelihoods[0]
    assert L.dist == dist and type(L.psi) is type(ref.likelihoods[0].psi)
    same_density(oracle(m), oracle(ref), m, ref, spread=0.5)
    # and it lowers: psi block one past the predictor's terms
    low = ir.lower(ir.fuse_design_columns(m))
    assert low.liks[0]["nu"] == (2.0 if psi_kind == "logit" else 0.0) and len(low.liks[0]["psi"]) == (2 if psi_kind == "logit" else 1)


def test_zip_with_a_logit_linear_psi_lowers_to_a_logit_block(fake_pytensor):
    """ZeroInflatedPoisson("y", psi=invlogit(Z @ g), mu=exp(X @ b)) -> zero_inflated_poisson with the logit block."""
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(1)
    N = 30
    X, Z = rng.standard_normal((N, 3)), rng.standard_normal((N, 2))
    M = FakeModel("zip")
    b = M.free(rv("NormalRV", "b", Constant(0.0), Constant(1.0)), 3)
    gm = M.free(rv("NormalRV", "g", Constant(0.0), Constant(1.0)), 2)
    psi = elem("Sigmoid", apply(Dot(), SharedVariable(Z), gm))
    y = rng.poisson(1.5, N).astype(np.float64)
    y[:10] = 0.0
    M.observe(rv("MixtureRV", "y", weights(psi), dirac(), rv("PoissonRV", None, elem("Exp", apply(Dot(), SharedVariable(X), b)))), y)
    m = ir.fuse_design_columns(from_pymc(M))
    L = m.likelihoods[0]
    assert L.dist == "zero_inflated_poisson" and isinstance(L.psi, ir.Linear)
    assert len(L.psi.terms) == 1 and ir.is_design(L.psi.terms[0]) and np.array_equal(L.psi.terms[0].coef, Z)
    low = ir.lower(m)
    assert low.liks[0]["nu"] == 1.0 and low.liks[0]["psi"][0]["n_cols"] == 2


def _refused(M_builder, match):
    from pymc_b200 import from_pymc

    M = M_builder()
    with pytest.raises(NotImplementedError, match=match):
        from_pymc(M)


def _base(N=12):
    rng = np.random.default_rng(2)
    M = FakeModel("bad")
    b = M.free(rv("NormalRV", "b", Constant(0.0), Constant(1.0)), 1)
    return M, bcast(b), rng.integers(0, 3, N).astype(np.float64), N


def test_other_mixtures_and_forms_of_psi_are_refused_by_name(fake_pytensor):
    def hurdle_lognormal():
        M, eta, y, N = _base()
        M.observe(rv("_HurdleRV", "y", weights(Constant(0.6)), dirac(),
                     rv("LogNormalRV", None, eta, Constant(1.0))), y + 0.5 * (y > 0))
        return M

    def normal_mixture():
        M, eta, y, N = _base()
        M.observe(rv("MixtureRV", "y", weights(Constant(0.6)), rv("NormalRV", None, eta, Constant(1.0)),
                     rv("NormalRV", None, eta, Constant(2.0))), y)
        return M

    def zi_gamma():
        M, eta, y, N = _base()
        M.observe(rv("MixtureRV", "y", weights(Constant(0.6)), dirac(),
                     rv("GammaRV", None, Constant(2.0), elem("Reciprocal", elem("TrueDiv", Constant(2.0), elem("Exp", eta))))), y)
        return M

    def vector_psi():
        M, eta, y, N = _base()
        p = M.free(rv("BetaRV", "p", Constant(2.0), Constant(2.0)), N, LogOddsTransform(), suffix="_logodds__")
        M.observe(rv("MixtureRV", "y", weights(p), dirac(), rv("PoissonRV", None, elem("Exp", eta))), y)
        return M

    def per_obs_psi():
        M, eta, y, N = _base()
        M.observe(rv("MixtureRV", "y", weights(Constant(np.full(N, 0.4))), dirac(), rv("PoissonRV", None, elem("Exp", eta))), y)
        return M

    def exp_psi():
        M, eta, y, N = _base()
        M.observe(rv("MixtureRV", "y", weights(elem("Exp", eta)), dirac(), rv("PoissonRV", None, elem("Exp", eta))), y)
        return M

    def weights_not_one_minus():
        M, eta, y, N = _base()
        w = apply(Join(), Constant(-1), bcast(Constant(0.5)), bcast(Constant(0.3)))
        M.observe(rv("MixtureRV", "y", w, dirac(), rv("PoissonRV", None, elem("Exp", eta))), y)
        return M

    def hurdle_untruncated_poisson():
        M, eta, y, N = _base()
        M.observe(rv("_HurdleRV", "y", weights(Constant(0.6)), dirac(), rv("PoissonRV", None, elem("Exp", eta))), y)
        return M

    _refused(hurdle_lognormal, "HurdleLogNormal is outside the closed set")
    _refused(normal_mixture, "pm.Mixture / pm.NormalMixture is outside the closed set")
    _refused(zi_gamma, "GammaRV component is outside the closed set")
    _refused(vector_psi, "vector psi variable")
    _refused(per_obs_psi, "per-observation constant psi")
    _refused(exp_psi, "stack\\(\\[1 - psi, psi\\]\\)")
    _refused(weights_not_one_minus, "stack\\(\\[1 - psi, psi\\]\\)")
    _refused(hurdle_untruncated_poisson, "PoissonRV component is outside the closed set")


def test_psi_of_one_is_refused_with_the_plain_likelihood_named(fake_pytensor):
    from pymc_b200 import from_pymc

    M, eta, y, N = _base()
    M.observe(rv("MixtureRV", "y", weights(Constant(1.0)), dirac(), rv("PoissonRV", None, elem("Exp", eta))), y)
    with pytest.raises(ValueError, match="write the plain likelihood"):
        from_pymc(M)
