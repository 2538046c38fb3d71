"""CPU: ``from_pymc`` on a STAND-IN graph.  PyMC / PyTensor are not importable in the build image (SURVEY 8c), so
tests/test_frontend.py (the real thing, under ``importorskip("pymc")``) never runs here.  This file drives the same lowering
code with a minimal imitation of the objects it walks -- variables with ``owner.op`` / ``owner.inputs``, RV ops named like
PyTensor's (``NormalRV``, ``HalfCauchyRV``), ``Elemwise`` with a ``scalar_op``, ``DimShuffle``, ``AdvancedSubtensor1``, ``Dot``,
``Constant`` -- wired into ``sys.modules`` for the duration of a test, builds the Eight Schools, Radon and hierarchical
logistic models as such graphs, and checks that the ModelIR that comes out has the log-density and gradient of the
hand-derived restatements (oracle/logp_numpy.py) and routes to the hand-specialised kernels."""
import sys
import types

import numpy as np
import pytest


# ---- the imitation graph ---------------------------------------------------------------------------------------------------
class Variable:
    def __init__(self, name=None, owner=None):
        self.name, self.owner = name, owner

    def __repr__(self):
        return f"<{type(self).__name__} {self.name}>"


class Constant(Variable):
    def __init__(self, data):
        super().__init__()
        self.data = np.asarray(data)


class SharedVariable(Variable):
    def __init__(self, value):
        super().__init__()
        self._v = np.asarray(value)

    def get_value(self):
        return self._v


class Apply:
    def __init__(self, op, inputs):
        self.op, self.inputs = op, list(inputs)


class DimShuffle:
    pass


class Elemwise:
    def __init__(self, scalar_op):
        self.scalar_op = scalar_op


class Dot:
    pass


class Join:
    pass


class Subtensor:
    pass


class AdvancedSubtensor(Subtensor):
    pass


class AdvancedSubtensor1(Subtensor):
    pass


def _scalar(name):
    return type(name, (), {})()


def apply(op, *inputs, name=None):
    return Variable(name, Apply(op, inputs))


def elem(kind, *inputs):
    return apply(Elemwise(_scalar(kind)), *inputs)


def bcast(x):
    return apply(DimShuffle(), x)


def rv(op_name, name, *params):
    op = type(op_name, (), {"dist_params": lambda self, node: node.inputs[2:]})()
    return apply(op, Variable("rng"), Constant(np.array([])), *params, name=name)


class LogTransform:
    pass


class FakeModel:
    def __init__(self, name="model"):
        self.name, self.free_RVs, self.observed_RVs = name, [], []
        self.rvs_to_values, self.rvs_to_transforms, self._ip = {}, {}, {}

    def free(self, r, size, transform=None, initial=None, suffix=None):
        """suffix: what PyMC appends to the value variable's name; "_log__" under a transform unless given."""
        vname = r.name + (suffix if suffix is not None else "_log__" if transform is not None else "")
        self.free_RVs.append(r)
        self.rvs_to_values[r] = Variable(vname)
        self.rvs_to_transforms[r] = transform
        self._ip[vname] = np.zeros(size) if initial is None else np.asarray(initial, dtype=float)
        return r

    def observe(self, r, data):
        self.observed_RVs.append(r)
        self.rvs_to_values[r] = Constant(data)
        return r

    def initial_point(self):
        return dict(self._ip)


@pytest.fixture
def fake_pytensor(monkeypatch):
    """pytensor / pymc module shells exposing the imitation classes where frontend.py imports them from."""
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__b200_stub__ = True
        monkeypatch.setitem(sys.modules, name, m)
        return m

    mod("pytensor")
    mod("pytensor.graph")
    mod("pytensor.graph.basic", Constant=Constant, Variable=Variable)
    mod("pytensor.compile")
    mod("pytensor.compile.sharedvalue", SharedVariable=SharedVariable)
    mod("pytensor.tensor")
    mod("pytensor.tensor.elemwise", DimShuffle=DimShuffle, Elemwise=Elemwise)
    mod("pytensor.tensor.math", Dot=Dot)
    mod("pytensor.tensor.subtensor", AdvancedSubtensor=AdvancedSubtensor, AdvancedSubtensor1=AdvancedSubtensor1, Subtensor=Subtensor)
    mod("pymc")
    mod("pymc.pytensorf")  # no constant_fold: frontend._const_value falls back to "not a constant"
    yield


def _same_density(m, f_ref, n, seed=0):
    from oracle import ir_numpy

    g = ir_numpy.make_logp(m)
    rng = np.random.default_rng(seed)
    for _ in range(4):
        q = m.initial_point() + rng.uniform(-0.7, 0.7, n)
        lp, dlp = g(q)
        lp_ref, dlp_ref = f_ref(q)
        assert abs(lp - lp_ref) <= 1e-11 * max(1.0, abs(lp_ref))
        np.testing.assert_allclose(dlp, dlp_ref, rtol=1e-10, atol=1e-10)


def same_density(f, g, m, ref, *, spread, seed=0):
    """m, which from_pymc made, against the hand-built IR ref: the same value variables and transforms, and the same
    log-density and gradient (f of m, g of ref, the caller's oracle) at four points around ref's initial point."""
    assert m.n == ref.n and [v.name for v in m.vars] == [v.name for v in ref.vars]
    assert [v.transform for v in m.vars] == [v.transform for v in ref.vars]
    rng = np.random.default_rng(seed)
    for _ in range(4):
        q = ref.initial_point() + rng.uniform(-spread, spread, ref.n)
        (a, ga), (b, gb) = f(q), g(q)
        assert abs(a - b) <= 1e-12 * abs(b)
        np.testing.assert_allclose(ga, gb, rtol=1e-12, atol=1e-12)


def test_eight_schools_graph_lowers_to_the_reference_density(fake_pytensor):
    from oracle import logp_numpy
    from pymc_b200 import from_pymc, ir, models

    spec = models.eight_schools()
    y, s = spec.data["y"], spec.data["sigma"]
    M = FakeModel("eight_schools")
    mu = M.free(rv("NormalRV", "mu", Constant(0.0), Constant(5.0)), 1)
    tau = M.free(rv("HalfCauchyRV", "tau", Constant(0.0), Constant(5.0)), 1, LogTransform())
    theta = M.free(rv("NormalRV", "theta_t", Constant(0.0), Constant(1.0)), 8)
    loc = elem("Add", bcast(mu), elem("Mul", bcast(tau), theta))
    M.observe(rv("NormalRV", "y", loc, Constant(s)), y)
    m = from_pymc(M)
    assert [v.name for v in m.vars] == ["mu", "tau_log__", "theta_t"] and m.n == spec.n
    assert [v.transform for v in m.vars] == [None, "log", None]
    _same_density(m, logp_numpy.make_logp(spec), spec.n)
    assert ir.specialise(m) is not None  # routed to the hand-specialised Eight Schools kernel


def test_radon_graph_lowers_to_the_reference_density(fake_pytensor):
    from oracle import logp_numpy
    from pymc_b200 import from_pymc, ir, models

    spec = models.radon(60, 7, 5)
    county, floor, y = spec.data["county_idx"], spec.data["floor"], spec.data["y"]
    J = spec.meta["n_counties"]
    M = FakeModel("radon")
    S = Constant(100.0**2)
    mu_a = M.free(rv("NormalRV", "mu_a", Constant(0.0), S), 1)
    sigma_a = M.free(rv("HalfCauchyRV", "sigma_a", Constant(0.0), Constant(5.0)), 1, LogTransform())
    mu_b = M.free(rv("NormalRV", "mu_b", Constant(0.0), S), 1)
    sigma_b = M.free(rv("HalfCauchyRV", "sigma_b", Constant(0.0), Constant(5.0)), 1, LogTransform())
    a = M.free(rv("NormalRV", "a", Constant(0.0), Constant(1.0)), J)
    b = M.free(rv("NormalRV", "b", Constant(0.0), Constant(1.0)), J)
    eps = M.free(rv("HalfCauchyRV", "eps", Constant(0.0), Constant(5.0)), 1, LogTransform())
    idx = Constant(county.astype(np.int64))
    alpha = elem("Add", bcast(mu_a), elem("Mul", apply(AdvancedSubtensor1(), a, idx), bcast(sigma_a)))
    beta = elem("Add", bcast(mu_b), elem("Mul", apply(AdvancedSubtensor1(), b, idx), bcast(sigma_b)))
    loc = elem("Add", alpha, elem("Mul", beta, Constant(floor)))
    M.observe(rv("NormalRV", "radon", loc, bcast(eps)), y)
    m = from_pymc(M)
    assert m.n == spec.n and [v.name for v in m.vars][:4] == ["mu_a", "sigma_a_log__", "mu_b", "sigma_b_log__"]
    _same_density(m, logp_numpy.make_logp(spec), spec.n, seed=1)
    assert ir.specialise(m) is not None  # the benchmark model's shape: routed to the hand-specialised Radon kernel


def test_hierarchical_logistic_graph_with_dot_and_shared_data(fake_pytensor):
    """alpha[g] + X @ beta under Bernoulli(logit_p): indexing, a constant-matrix dot (held in a shared variable), a Normal prior
    whose parameters are scalar free RVs."""
    from scipy import stats as st

    from oracle import ir_numpy
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(2)
    N, G, K = 70, 5, 3
    g = rng.integers(0, G, N)
    X = rng.standard_normal((N, K))
    y = (rng.random(N) < 0.5).astype(float)
    M = FakeModel("hlogit")
    mu = M.free(rv("NormalRV", "mu", Constant(0.0), Constant(2.0)), 1)
    s = M.free(rv("HalfNormalRV", "s", Constant(0.0), Constant(1.0)), 1, LogTransform())
    alpha = M.free(rv("NormalRV", "alpha", bcast(mu), bcast(s)), G)
    beta = M.free(rv("NormalRV", "beta", Constant(0.0), Constant(2.5)), K)
    eta = elem("Add", apply(AdvancedSubtensor1(), alpha, Constant(g)), apply(Dot(), SharedVariable(X), beta))
    M.observe(rv("BernoulliRV", "y", elem("Sigmoid", eta)), y)
    m = from_pymc(M)
    assert m.likelihoods[0].dist == "bernoulli_logit" and len(m.likelihoods[0].terms) == 1 + K
    f = ir_numpy.make_logp(m)

    def ref(q):  # the density from scipy.stats compositions, in the value-variable order mu, s_log__, alpha, beta
        mu_, ls, al, be = q[0], q[1], q[2 : 2 + G], q[2 + G :]
        sd = np.exp(ls)
        e = al[g] + X @ be
        return (st.norm(0, 2).logpdf(mu_) + st.halfnorm(scale=1).logpdf(sd) + ls + st.norm(mu_, sd).logpdf(al).sum()
                + st.norm(0, 2.5).logpdf(be).sum() + np.sum(y * e - np.logaddexp(0.0, e)))

    q = m.initial_point() + rng.uniform(-0.5, 0.5, m.n)
    lp, dlp = f(q)
    assert abs(lp - ref(q)) <= 1e-10 * abs(ref(q))
    h = 1e-6
    num = np.array([(ref(q + h * np.eye(m.n)[i]) - ref(q - h * np.eye(m.n)[i])) / (2 * h) for i in range(m.n)])
    np.testing.assert_allclose(dlp, num, rtol=1e-5, atol=1e-6)


class IntervalTransform:
    def __init__(self, lo, hi):
        self._b = (lo, hi)

    def args_fn(self, *inputs):
        return self._b


def test_stochastic_volatility_graph_ar1_interval_and_log_variance_likelihood(fake_pytensor):
    """BASELINE config 4 as a PyMC graph: mu ~ Normal(0, 5), phi ~ Uniform(-1, 1) (interval transform), sigma ~ Exponential(10)
    (PyTensor's scale parametrisation), h ~ AR(rho=[phi], sigma, init_dist=Normal(0, 1)), y ~ Normal(0, exp((mu + h) / 2))."""
    from oracle import logp_numpy
    from pymc_b200 import from_pymc, models

    spec = models.stochvol(T=40, seed=4)
    y = spec.data["y"]
    T = len(y)
    M = FakeModel("stochvol")
    mu = M.free(rv("NormalRV", "mu", Constant(0.0), Constant(5.0)), 1)
    lo, hi = Constant(-1.0), Constant(1.0)
    phi = rv("UniformRV", "phi", lo, hi)
    M.free(phi, 1, IntervalTransform(lo, hi), suffix="_interval__")
    sigma = M.free(rv("ExponentialRV", "sigma", Constant(0.1)), 1, LogTransform(), initial=[np.log(0.1)])
    init = rv("NormalRV", "init", Constant(0.0), Constant(1.0))
    ar_op = type("AutoRegressiveRV", (), {"ar_order": 1, "constant_term": False,
                                          "dist_params": lambda self, node: node.inputs[2:]})()
    h = apply(ar_op, Variable("rng"), Constant(np.array([])), apply(DimShuffle(), phi), bcast(sigma), init, name="h")
    M.free(h, T)
    log_sd = elem("TrueDiv", elem("Add", bcast(mu), h), Constant(2.0))
    M.observe(rv("NormalRV", "y", Constant(0.0), elem("Exp", log_sd)), y)
    m = from_pymc(M)
    assert [v.name for v in m.vars] == ["mu", "phi_interval__", "sigma_log__", "h"] and m.n == spec.n
    assert m.vars[1].transform == "interval" and m.vars[1].bounds == (-1.0, 1.0)
    assert m.likelihoods[0].dist == "normal_logvar" and len(m.ar1) == 1
    _same_density(m, logp_numpy.make_logp(spec), spec.n, seed=3)


def test_deterministics_are_lowered_and_evaluated_from_the_draws(fake_pytensor):
    """pm.Deterministic("theta", mu + tau * theta_t): lowered to the same linear-predictor form, evaluated on the host from the
    constrained draws, never part of logp."""
    from pymc_b200 import from_pymc, models

    spec = models.eight_schools()
    M = FakeModel("eight_schools")
    mu = M.free(rv("NormalRV", "mu", Constant(0.0), Constant(5.0)), 1)
    tau = M.free(rv("HalfCauchyRV", "tau", Constant(0.0), Constant(5.0)), 1, LogTransform())
    theta_t = M.free(rv("NormalRV", "theta_t", Constant(0.0), Constant(1.0)), 8)
    loc = elem("Add", bcast(mu), elem("Mul", bcast(tau), theta_t))
    M.observe(rv("NormalRV", "y", loc, Constant(spec.data["sigma"])), spec.data["y"])
    theta = apply(type("Identity", (), {})(), loc, name="theta")
    theta.type = types.SimpleNamespace(shape=(8,))
    half = elem("TrueDiv", bcast(mu), Constant(2.0))
    half.name, half.type = "half_mu", types.SimpleNamespace(shape=())
    M.deterministics = [theta, half]
    m = from_pymc(M)
    assert [d.name for d in m.deterministics] == ["theta", "half_mu"] and [d.size for d in m.deterministics] == [8, 1]
    q = m.initial_point() + np.random.default_rng(0).normal(size=(2, 3, m.n))
    c = m.constrain(q)
    d = m.eval_deterministics(c)
    np.testing.assert_allclose(d["theta"], c["mu"][..., None] + c["tau"][..., None] * c["theta_t"], rtol=1e-14)
    np.testing.assert_allclose(d["half_mu"], 0.5 * c["mu"], rtol=1e-14)
    unknown = elem("Add", bcast(mu), theta_t)
    unknown.name, unknown.type = "u", types.SimpleNamespace(shape=(None,))
    M.deterministics = [unknown]
    with pytest.raises(NotImplementedError, match="statically"):
        from_pymc(M)


def test_graphs_outside_the_closed_set_are_refused(fake_pytensor):
    from pymc_b200 import from_pymc

    M = FakeModel()
    M.free(rv("WeibullRV", "w", Constant(1.0), Constant(2.0)), 1, LogTransform())
    with pytest.raises(NotImplementedError, match="outside the closed set"):
        from_pymc(M)
    M2 = FakeModel()
    x = M2.free(rv("NormalRV", "x", Constant(0.0), Constant(1.0)), 4)
    M2.observe(rv("NormalRV", "y", elem("Tanh", x), Constant(1.0)), np.zeros(4))
    with pytest.raises(NotImplementedError, match="linear predictor"):
        from_pymc(M2)
