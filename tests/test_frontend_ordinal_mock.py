"""CPU: ``from_pymc`` on imitation graphs (tests/test_frontend_mock.py's stand-ins) of ordinal regressions.

pm.OrderedLogistic(eta, cutpoints) and pm.OrderedProbit(eta, cutpoints, sigma) build a Categorical whose p is
``compute_p`` (pymc/distributions/discrete.py:1312-1326: differences of the concatenation [0, sigmoid(cutpoints -
eta[:, None]), 1]; :1416-1432: exp of the concatenation of normal_lccdf / log_diff_normal_cdf / normal_lcdf of
eta[:, None] - cutpoints, each standardising as (x - 0) / sigma, dist_math.py:126-182), with the ``{name}_probs``
Deterministic between them when compute_p=True.  Each graph must lower to an IR with the density of the hand-built IR and
record the probabilities; the Ordered transform maps to "ordered" / "ordered_positive"; other Categoricals, descending and
chained transforms and unordered vector cutpoints are refused by name.  A real-PyMC test runs where PyMC is importable."""
import numpy as np
import pytest
from scipy import special, stats
from test_frontend_mock import Constant, FakeModel, LogTransform, SharedVariable, apply, bcast, elem, fake_pytensor, rv  # noqa: F401
from test_frontend_mock import AdvancedSubtensor1, Dot, Join, Subtensor, same_density
from test_ir_ordinal import oracle

from pymc_b200 import ir


def _op(name):
    return type(name, (), {})()


def ordered(positive=False, ascending=True):
    return type("Ordered", (), {"positive": positive, "ascending": ascending})()


def _sub(x):
    return apply(Subtensor(), x)


def logistic_p(eta, cut):
    pa = elem("Sigmoid", elem("Sub", bcast(cut), bcast(eta)))
    cum = apply(Join(), Constant(-1), bcast(Constant(0.0)), pa, bcast(Constant(1.0)))
    return elem("Sub", _sub(cum), _sub(cum))


def probit_p(eta, cut, sigma):
    probits = elem("Sub", bcast(eta), bcast(cut))
    z = lambda x, s: elem("TrueDiv", elem("Sub", x, Constant(0.0)), s)  # noqa: E731
    r2 = Constant(np.sqrt(2.0))
    lccdf = elem("Switch", elem("GT", z(_sub(probits), sigma), Constant(1.0)),
                 elem("Log", elem("Erfcx", elem("TrueDiv", z(_sub(probits), sigma), r2))),
                 elem("Log1p", elem("Erfc", z(_sub(probits), sigma))))
    x, y = (elem("TrueDiv", z(_sub(probits), bcast(sigma)), r2) for _ in range(2))
    ldiff = elem("Add", Constant(np.log(0.5)), elem("Log", elem("Sub", elem("Erf", x), elem("Erf", y))))
    lcdf = elem("Log1p", elem("Erfc", z(_sub(probits), sigma)))
    return elem("Exp", apply(Join(), Constant(-1), bcast(lccdf), ldiff, bcast(lcdf)))


def _model(link, compute_p=True, sigma="const", positive=False, seed=3, N=40, K=5, cut_transform="ordered"):
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 4, N).astype(np.int32)
    X = rng.standard_normal((N, 2))
    y = rng.integers(0, K, N).astype(np.float64)
    mu_c = np.linspace(-2.0, 2.0, K - 1)
    M = FakeModel("ordinal")
    a = M.free(rv("NormalRV", "a", Constant(0.0), Constant(1.0)), 4)
    beta = M.free(rv("NormalRV", "beta", Constant(0.0), Constant(1.0)), 2)
    tr = ordered(positive) if cut_transform == "ordered" else cut_transform
    z0 = np.concatenate([[0.0 if positive else -2.0], np.log(np.diff(mu_c))])
    cut = M.free(rv("NormalRV", "cutpoints", Constant(mu_c), Constant(5.0)), K - 1, tr, initial=z0,
                 suffix="_ordered__" if type(tr).__name__ == "Ordered" else None)
    vars_ = [ir.Var("a", "a", 4), ir.Var("beta", "beta", 2),
             ir.Var("cutpoints_ordered__", "cutpoints", K - 1, "ordered_positive" if positive else "ordered")]
    priors = [ir.Prior("normal", "a", (0.0, 1.0)), ir.Prior("normal", "beta", (0.0, 1.0)),
              ir.Prior("normal", "cutpoints_ordered__", (ir.Linear([ir.Term([], coef=mu_c)]), 5.0))]
    eta = elem("Add", apply(AdvancedSubtensor1(), a, Constant(g)), apply(Dot(), SharedVariable(X), beta))
    s_ir = None
    if link == "logistic":
        p = logistic_p(eta, cut)
    else:
        if sigma == "var":
            s = M.free(rv("HalfNormalRV", "sigma", Constant(0.0), Constant(1.0)), 1, LogTransform())
            vars_.append(ir.Var("sigma_log__", "sigma", 1, "log"))
            priors.append(ir.Prior("halfnormal", "sigma_log__", (1.0,)))
            s_ir = ir.Ref("sigma_log__")
        else:
            s, s_ir = Constant(1.0), 1.0
        p = probit_p(eta, cut, s)
    if compute_p:
        p = apply(_op("Identity"), p, name="y_probs")
        M.deterministics = [p]
    M.observe(rv("CategoricalRV", "y", p), y)
    terms = [ir.Term([("a", g)])] + [ir.Term([("beta", np.full(N, k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(2)]
    ref = ir.ModelIR(vars=vars_, priors=priors,
                     likelihoods=[ir.Likelihood(f"ordered_{link}", y, terms, sigma=s_ir, cutpoints=ir.Ref("cutpoints_ordered__"))])
    return M, ref


def _numpy_probs(link, eta, c, s=1.0):
    """compute_p restated in probability space (discrete.py:1312-1326, :1416-1432)"""
    cc = np.concatenate([[-np.inf], c, [np.inf]])
    if link == "logistic":
        cum = special.expit(cc[None, :] - eta[:, None])
    else:
        cum = stats.norm.cdf((cc[None, :] - eta[:, None]) / s)
    return cum[:, 1:] - cum[:, :-1]


@pytest.mark.parametrize("compute_p", [True, False])
@pytest.mark.parametrize("link,sigma", [("logistic", None), ("probit", "const"), ("probit", "var")])
def test_ordinal_graphs_lower_to_the_ordinal_likelihoods(fake_pytensor, link, sigma, compute_p):
    from pymc_b200 import from_pymc

    M, ref = _model(link, compute_p, sigma)
    m = from_pymc(M)
    L = m.likelihoods[0]
    assert L.dist == f"ordered_{link}" and L.cutpoints == ir.Ref("cutpoints_ordered__")
    assert L.sigma == ref.likelihoods[0].sigma
    same_density(oracle(m), oracle(ref), m, ref, spread=0.5)
    if not compute_p:
        assert m.deterministics == []
        return
    (d,) = m.deterministics
    assert d.name == "y_probs" and d.probs_of == "y" and d.size == 40 * 5
    q = ref.initial_point() + np.random.default_rng(1).uniform(-0.5, 0.5, (3, 2, ref.n))
    post = m.constrain(q)
    probs = m.eval_deterministics(post)["y_probs"]
    assert probs.shape == (3, 2, 40, 5)
    np.testing.assert_allclose(probs.sum(-1), 1.0, rtol=1e-13)
    f = oracle(m)
    for ix in np.ndindex(3, 2):
        x, _ = f.constrained(q[ix])
        s = 1.0 if link == "logistic" else f.scale(L, x)[0]
        want = _numpy_probs(link, f.eta(L, x)[0], f.cutpoints(L, x), s)
        np.testing.assert_allclose(probs[ix], want, rtol=1e-12, atol=1e-15)


def test_ordered_positive_transform_maps_to_ordered_positive(fake_pytensor):
    from pymc_b200 import from_pymc

    M, ref = _model("logistic", positive=True)
    m = from_pymc(M)
    assert m.var("cutpoints").transform == "ordered_positive"
    same_density(oracle(m), oracle(ref), m, ref, spread=0.5)


def test_other_categoricals_and_transforms_are_refused_by_name(fake_pytensor):
    from pymc_b200 import from_pymc

    y = np.array([0.0, 1.0, 2.0])

    def plain(p):
        M = FakeModel("cat")
        M.free(rv("NormalRV", "b", Constant(0.0), Constant(1.0)), 1)
        M.observe(rv("CategoricalRV", "y", p), y)
        return M

    for what, M in [
        ("Categorical: only", plain(Constant(np.array([0.2, 0.3, 0.5])))),
        ("Categorical: only", plain(apply(_op("Softmax"), bcast(Constant(np.zeros(3)))))),
        ("Categorical: only", plain(elem("Sub", Constant(np.ones(3)), Constant(np.zeros(3))))),
    ]:
        with pytest.raises(NotImplementedError, match=what):
            from_pymc(M)
    with pytest.raises(NotImplementedError, match=r"Ordered\(ascending=False\)"):
        from_pymc(_model("logistic", cut_transform=ordered(ascending=False))[0])
    with pytest.raises(NotImplementedError, match=r"Chain\(\[\.\.\.\]\)"):
        from_pymc(_model("logistic", cut_transform=_op("Chain"))[0])
    with pytest.raises(NotImplementedError, match="unordered vector cutpoints"):
        from_pymc(_model("probit", cut_transform=None)[0])


def test_real_pymc_ordered_logistic_and_probit_lower_to_the_oracle_density():
    pm = pytest.importorskip("pymc")
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(5)
    N, K = 60, 4
    X = rng.standard_normal((N, 2))
    y = rng.integers(0, K, N)
    for link in ("logistic", "probit"):
        with pm.Model() as model:
            beta = pm.Normal("beta", 0.0, 1.0, shape=2)
            cut = pm.Normal("cutpoints", mu=np.linspace(-2, 2, K - 1), sigma=5, shape=K - 1,
                            transform=pm.distributions.transforms.ordered)
            eta = pm.math.dot(X, beta)
            if link == "logistic":
                pm.OrderedLogistic("y", eta=eta, cutpoints=cut, observed=y)
            else:
                pm.OrderedProbit("y", eta=eta, cutpoints=cut, sigma=1.0, observed=y)
        m = from_pymc(model)
        assert m.likelihoods[0].dist == f"ordered_{link}" and m.var("cutpoints").transform == "ordered"
        f = oracle(m)
        lp_fn = model.compile_logp()
        q = m.initial_point()
        ip = model.initial_point()
        want = float(lp_fn(ip))
        assert abs(f(q)[0] - want) <= 1e-9 * max(1.0, abs(want))
        assert [d.name for d in m.deterministics] == ["y_probs"]
