"""Design-matrix terms of the model IR: ``Term([(beta, None)], coef=X)`` with X [N][K] adds X @ beta to a linear predictor.

CPU: validation, ``fuse_design_columns`` (the column form ``from_pymc`` and the builders write, turned into design terms),
lowering, Deterministics, constant data and ``specialise``.  GPU: the generic device function and the pointwise kernel
against a NumPy evaluation, bit-reproducibility, fixed-step NUTS against the oracle sampler, and the C ABI's refusals.

The NumPy evaluation of a design term (``design_logp``) uses the oracle unchanged: each design term becomes an elementwise
offset variable u = X @ x of the likelihood's length, whose oracle gradient is d logp / d eta = r, and X.T @ r is the
design variable's share of the gradient.
"""
from __future__ import annotations

import copy
import dataclasses
import re

import numpy as np
import pytest
from b200_helpers import fixed_step_against_oracle, logp_at_both_team_shapes, random_dense_cov, refusal_after_edit
from test_frontend_mock import (AdvancedSubtensor1, Constant, Dot, FakeModel, LogTransform, SharedVariable, apply, bcast,
                                elem, fake_pytensor, rv)  # noqa: F401
from test_ir_closed_set import GRAD_TOL, LP_TOL, scipy_loglik

from pymc_b200 import ir
from pymc_b200.ir import Deterministic, Likelihood, ModelIR, Prior, Ref, Term, Var


# ------------------------------------------------------------------------------------------------------------------------
# NumPy evaluation of models with design terms
# ------------------------------------------------------------------------------------------------------------------------
def _constrained(m, q):
    c, off = m.constrain(q), m.offsets()
    x, dxdq = np.empty(m.n), np.ones(m.n)
    for v in m.vars:
        s = slice(off[v.name], off[v.name] + v.size)
        x[s] = np.ravel(c[v.rv_name])
        if v.transform == "log":
            dxdq[s] = x[s]
        elif v.transform == "interval":
            lo, hi = v.bounds
            sg = (x[s] - lo) / (hi - lo)
            dxdq[s] = (hi - lo) * sg * (1.0 - sg)
    return x, dxdq


class DesignLogp:
    """q -> (logp, dlogp) of a model whose likelihoods may hold design terms."""

    def __init__(self, m: ModelIR):
        from oracle import ir_numpy_families

        m.validate()
        self.m, self.off = m, m.offsets()
        self.design = []  # (X, variable slice, offset slot slice in the augmented q)
        aug = dataclasses.replace(m, vars=list(m.vars), likelihoods=[], deterministics=[])
        n_aug = m.n
        for L in m.likelihoods:
            terms = []
            for t in L.terms:
                if ir.is_design(t):
                    v = m.var(t.factors[0][0])
                    name = f"design_offset{len(self.design)}"
                    aug.vars.append(Var(name, name, len(L.y)))
                    self.design.append((np.asarray(t.coef, dtype=np.float64), slice(self.off[v.name], self.off[v.name] + v.size),
                                        slice(n_aug, n_aug + len(L.y))))
                    n_aug += len(L.y)
                    terms.append(Term([(name, None)]))
                else:
                    terms.append(t)
            aug.likelihoods.append(dataclasses.replace(L, terms=terms))
        self.base = ir_numpy_families.make_logp(aug)

    def __call__(self, q):
        q = np.asarray(q, dtype=np.float64)
        x, dxdq = _constrained(self.m, q)
        u = [X @ x[vs] for X, vs, _ in self.design]
        lp, ga = self.base(np.concatenate([q] + u))
        g = ga[: self.m.n].copy()
        for X, vs, us in self.design:
            g[vs] += (X.T @ ga[us]) * dxdq[vs]
        return lp, g


def design_logp(m):
    return DesignLogp(m)


def eta_of(m, L, x):
    """The linear predictor of likelihood L at the constrained values x."""
    off, N = m.offsets(), len(L.y)
    eta = np.zeros(N)
    for t in L.terms:
        if ir.is_design(t):
            v = m.var(t.factors[0][0])
            eta = eta + np.asarray(t.coef) @ x[off[v.name] : off[v.name] + v.size]
            continue
        term = np.ones(N) if t.coef is None else np.broadcast_to(np.asarray(t.coef, dtype=np.float64), (N,))
        for vn, idx in t.factors:
            v = m.var(vn)
            xv = x[off[v.name] : off[v.name] + v.size]
            term = term * (xv[idx] if idx is not None else (xv[0] if v.size == 1 else xv))
        eta = eta + term
    return eta


def lik_param(m, L, x):
    par = L.trials if L.dist == "binomial_logit" else (L.alpha if L.alpha is not None else L.sigma)
    if isinstance(par, Ref):
        return x[m.offsets()[m.var(par.var).name]]
    return 1.0 if par is None else np.asarray(par, dtype=np.float64)


def pieces_scale(m, q, lp):
    """sum |pieces| of the log density at q: every observation's log-likelihood, plus the rest as one piece."""
    x, _ = _constrained(m, q)
    S, ll_sum = 0.0, 0.0
    for L in m.likelihoods:
        ll = scipy_loglik(L.dist, np.asarray(L.y, dtype=np.float64), eta_of(m, L, x), lik_param(m, L, x), L.nu)
        S += np.sum(np.abs(ll))
        ll_sum += np.sum(ll)
    return S + abs(lp - ll_sum)


# ------------------------------------------------------------------------------------------------------------------------
# models
# ------------------------------------------------------------------------------------------------------------------------
FAMILIES = ["normal", "studentt", "bernoulli_logit", "poisson_log", "normal_logvar", "binomial_logit", "negative_binomial_log",
            "gamma_log"]


def _observe(dist, eta, rng):
    """(y, likelihood keyword arguments, extra variables, extra priors) of one family at linear predictor eta."""
    N = len(eta)
    if dist in ("normal", "studentt"):
        kw = dict(sigma=Ref("sigma_log__"), nu=4.0 if dist == "studentt" else 0.0)
        return (eta + 0.5 * rng.standard_normal(N), kw, [Var("sigma_log__", "sigma", 1, "log", initial=np.log(0.5))],
                [Prior("halfnormal", "sigma_log__", (1.0,))])
    if dist == "bernoulli_logit":
        return (rng.random(N) < 1.0 / (1.0 + np.exp(-eta))).astype(np.float64), {}, [], []
    if dist == "poisson_log":
        return rng.poisson(np.exp(eta)).astype(np.float64), {}, [], []
    if dist == "normal_logvar":
        return rng.standard_normal(N) * np.exp(eta / 2), {}, [], []
    if dist == "binomial_logit":
        n = rng.integers(1, 12, N).astype(np.float64)
        return rng.binomial(n.astype(np.int64), 1.0 / (1.0 + np.exp(-eta))).astype(np.float64), dict(trials=n), [], []
    extra = [Var("alpha_log__", "alpha", 1, "log", initial=np.log(2.0))], [Prior("exponential", "alpha_log__", (0.5,))]
    if dist == "negative_binomial_log":
        mu = np.exp(eta)
        return rng.negative_binomial(2.0, 2.0 / (mu + 2.0)).astype(np.float64), dict(alpha=Ref("alpha_log__")), *extra
    return rng.gamma(2.0, np.exp(eta) / 2.0), dict(alpha=Ref("alpha_log__")), *extra


def design_model(dist, N, K, seed=0, *, group=0, log_beta=False):
    """b0 + X @ beta (+ a[g] with `group` groups) under likelihood `dist`; beta ~ Normal(0, 1), or HalfNormal(1) under a log
    transform.  X is scaled so that eta stays of order one for any K."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, K)) / np.sqrt(K)
    beta_v = Var("beta_log__", "beta", K, "log") if log_beta else Var("beta", "beta", K)
    vars_ = [Var("b0", "b0", 1), beta_v]
    priors = [Prior("normal", "b0", (0.0, 1.0)), Prior("halfnormal" if log_beta else "normal", beta_v.name,
                                                      (1.0,) if log_beta else (0.0, 1.0))]
    terms = [Term([("b0", None)]), Term([(beta_v.name, None)], coef=X)]
    eta = 0.2 + X @ (np.abs(rng.normal(0.0, 1.0, K)) if log_beta else rng.normal(0.0, 1.0, K))
    if group:
        g = rng.integers(0, group, N).astype(np.int32)
        vars_.append(Var("a", "a", group))
        priors.append(Prior("normal", "a", (0.0, 0.5)))
        terms.append(Term([("a", g)]))
        eta = eta + rng.normal(0.0, 0.5, group)[g]
    y, kw, xv, xp = _observe(dist, eta, rng)
    return ModelIR(name=f"design-{dist}-N{N}-K{K}", vars=vars_ + xv, priors=priors + xp,
                   likelihoods=[Likelihood(dist, y, terms, **kw)])


def two_likelihoods_model(K=40, seed=3):
    """beta enters a Normal likelihood and a Bernoulli likelihood, each through its own X."""
    rng = np.random.default_rng(seed)
    X1, X2 = rng.standard_normal((60, K)) / np.sqrt(K), rng.standard_normal((25, K)) / np.sqrt(K)
    b = rng.normal(0.0, 1.0, K)
    y1 = X1 @ b + 0.3 * rng.standard_normal(60)
    y2 = (rng.random(25) < 1.0 / (1.0 + np.exp(-X2 @ b))).astype(np.float64)
    return ModelIR(name="design-two-likelihoods",
                   vars=[Var("beta", "beta", K), Var("sigma_log__", "sigma", 1, "log")],
                   priors=[Prior("normal", "beta", (0.0, 1.0)), Prior("halfnormal", "sigma_log__", (1.0,))],
                   likelihoods=[Likelihood("normal", y1, [Term([("beta", None)], coef=X1)], sigma=Ref("sigma_log__"), name="y1"),
                                Likelihood("bernoulli_logit", y2, [Term([("beta", None)], coef=X2)], name="y2")])


def two_design_terms_model(K=33, K2=7, N=90, seed=4):
    """Three design terms in one likelihood: on beta, on c, and on beta again."""
    rng = np.random.default_rng(seed)
    X1, X2, X3 = (rng.standard_normal((N, k)) / np.sqrt(k) for k in (K, K2, K))
    y = rng.poisson(np.exp(0.3 + 0.3 * rng.standard_normal(N))).astype(np.float64)
    return ModelIR(name="design-three-terms", vars=[Var("beta", "beta", K), Var("c", "c", K2)],
                   priors=[Prior("normal", "beta", (0.0, 1.0)), Prior("normal", "c", (0.0, 1.0))],
                   likelihoods=[Likelihood("poisson_log", y, [Term([("beta", None)], coef=X1), Term([("c", None)], coef=X2),
                                                               Term([("beta", None)], coef=X3)])])


def as_columns(m):
    """The column form of a model with design terms: one term per column k, beta[k] gathered by a constant index."""
    out = copy.deepcopy(m)
    for L in out.likelihoods:
        N, terms = len(L.y), []
        for t in L.terms:
            if ir.is_design(t):
                X = np.asarray(t.coef)
                terms += [Term([(t.factors[0][0], np.full(N, k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(X.shape[1])]
            else:
                terms.append(t)
        L.terms = terms
    return out


def _points(m, P, seed, spread=0.5):
    return m.initial_point() + np.random.default_rng(seed).uniform(-spread, spread, (P, m.n))


def _terms_equal(a, b):
    if len(a) != len(b):
        return False
    for s, t in zip(a, b):
        if [f[0] for f in s.factors] != [f[0] for f in t.factors]:
            return False
        for (_, i1), (_, i2) in zip(s.factors, t.factors):
            if (i1 is None) != (i2 is None) or (i1 is not None and not np.array_equal(i1, i2)):
                return False
        if (s.coef is None) != (t.coef is None) or (s.coef is not None and not np.array_equal(s.coef, t.coef)):
            return False
    return True


# ------------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------------
def test_validate_accepts_a_design_term_and_refuses_malformed_ones():
    m = design_model("normal", 20, 5)
    m.validate()
    X = m.likelihoods[0].terms[1].coef

    def edited(term):
        e = copy.deepcopy(m)
        e.likelihoods[0].terms[1] = term
        return e

    for term, msg in [
        (Term([("beta", None)], coef=X[:, :4]), r"X must have shape \(N, size of the variable\)"),
        (Term([("beta", None)], coef=X[:19]), r"X must have shape \(N, size of the variable\)"),
        (Term([("b0", None)], coef=X), r"X must have shape \(N, size of the variable\)"),
        (Term([("beta", None), ("b0", None)], coef=X), "a design term has exactly one factor"),
        (Term([], coef=X), "a design term has exactly one factor"),
        (Term([("beta", np.zeros(20, dtype=np.int32))], coef=X), "a design term's factor takes no index"),
        (Term([("beta", None)], coef=np.where(np.arange(5) == 2, np.nan, X)), "X must be finite"),
        (Term([("beta", None)], coef=np.where(np.arange(5) == 2, np.inf, X)), "X must be finite"),
    ]:
        with pytest.raises(ValueError, match=msg):
            edited(term).validate()
        with pytest.raises(ValueError, match=msg):
            ir.lower(edited(term))


@pytest.mark.parametrize("builder,K", [(ir.varying_intercept_logistic_ir, 3), (ir.negative_binomial_ir, 2),
                                       (ir.gamma_regression_ir, 3)])
def test_fuse_design_columns_fuses_the_builders(builder, K):
    m = builder()
    before = copy.deepcopy(m)
    f = ir.fuse_design_columns(m)
    L0, L = m.likelihoods[0], f.likelihoods[0]
    first = next(j for j, t in enumerate(L0.terms) if t.factors[0][0] == "beta")
    assert len(L.terms) == len(L0.terms) - K + 1
    assert ir.is_design(L.terms[first]) and L.terms[first].factors == [("beta", None)]
    assert _terms_equal(L.terms[:first], L0.terms[:first])
    X = np.column_stack([t.coef for t in L0.terms if t.factors[0][0] == "beta"])
    assert np.array_equal(L.terms[first].coef, X)
    assert _terms_equal(m.likelihoods[0].terms, before.likelihoods[0].terms)  # the input is untouched
    f.validate()


def test_fuse_design_columns_leaves_everything_else_as_written():
    rng = np.random.default_rng(1)
    N, K = 30, 4
    X = rng.standard_normal((N, K))
    g = rng.integers(0, 3, N).astype(np.int32)
    col = lambda k, coef=True: Term([("beta", np.full(N, k, dtype=np.int32))], coef=X[:, k].copy() if coef else None)  # noqa: E731
    base = dict(vars=[Var("beta", "beta", K), Var("a", "a", 3), Var("s", "s", 1)],
                priors=[Prior("normal", "beta", (0.0, 1.0)), Prior("normal", "a", (0.0, 1.0)), Prior("normal", "s", (0.0, 1.0))])
    y = rng.standard_normal(N)
    cases = {
        "partial": [col(0), col(1), col(3)],
        "duplicated": [col(0), col(1), col(2), col(3), col(2)],
        "group effect": [Term([("a", g)]), Term([("s", None), ("a", g)])],
        "multi-factor": [Term([("s", None), ("beta", np.full(N, k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(K)],
        "varying index": [Term([("beta", g)], coef=X[:, 0].copy())] + [col(k) for k in range(1, K)],
    }
    for what, terms in cases.items():
        m = ModelIR(**copy.deepcopy(base), likelihoods=[Likelihood("normal", y, terms, sigma=1.0)],
                    deterministics=[Deterministic("d", N, [col(k) for k in range(K)])])
        f = ir.fuse_design_columns(m)
        assert _terms_equal(f.likelihoods[0].terms, m.likelihoods[0].terms), what
        assert _terms_equal(f.deterministics[0].terms, m.deterministics[0].terms), what
    # a run with scalar and missing coefficients fuses, in place of its first term, around other terms
    terms = [Term([("a", g)]), Term([("beta", np.full(N, 2, dtype=np.int32))], coef=0.5), col(0), Term([("s", None)]),
             Term([("beta", np.full(N, 1, dtype=np.int32))]), col(3)]
    m = ModelIR(**copy.deepcopy(base), likelihoods=[Likelihood("normal", y, terms, sigma=1.0)])
    f = ir.fuse_design_columns(m)
    T = f.likelihoods[0].terms
    assert len(T) == 3 and T[0] is not terms[0] and ir.is_design(T[1]) and T[2].factors == [("s", None)]
    want = X.copy()
    want[:, 2], want[:, 1] = 0.5, 1.0
    assert np.array_equal(T[1].coef, want)
    assert len(m.likelihoods[0].terms) == 6 and m.likelihoods[0].terms[1].coef == 0.5


def _oracle_same(a, b, Q):
    fa, fb = design_logp(a), design_logp(b)
    for q in Q:
        (la, ga), (lb, gb) = fa(q), fb(q)
        assert abs(la - lb) <= 1e-13 * abs(lb), (la, lb)
        assert np.max(np.abs(ga - gb)) <= 1e-13 * max(1.0, np.max(np.abs(gb)))


@pytest.mark.parametrize("builder", [ir.varying_intercept_logistic_ir, ir.negative_binomial_ir, ir.gamma_regression_ir])
def test_fused_builders_have_the_column_form_density(builder):
    from oracle import ir_numpy_families

    m = builder()
    f = ir.fuse_design_columns(m)
    Q = _points(m, 4, 2)
    _oracle_same(f, m, Q)
    col = ir_numpy_families.make_logp(m)  # the column form through the oracle alone
    for q in Q:
        (la, ga), (lb, gb) = design_logp(f)(q), col(q)
        assert abs(la - lb) <= 1e-13 * abs(lb) and np.max(np.abs(ga - gb)) <= 1e-13 * max(1.0, np.max(np.abs(gb)))


def test_design_models_equal_their_column_form_in_the_oracle():
    for m in [design_model("poisson_log", 50, 31, group=4), two_likelihoods_model(), two_design_terms_model(),
              design_model("gamma_log", 40, 9, log_beta=True)]:
        _oracle_same(m, as_columns(m), _points(m, 3, 5))
        f = ir.fuse_design_columns(as_columns(m))
        n_design = sum(ir.is_design(t) for L in f.likelihoods for t in L.terms)
        # beta's two runs in the three-term model form a duplicated run, which stays in column form; c's run fuses
        assert n_design == (1 if m.name == "design-three-terms" else sum(ir.is_design(t) for L in m.likelihoods for t in L.terms))
        _oracle_same(f, m, _points(m, 3, 6))


def test_the_frontend_dot_graph_fuses_to_the_same_density(fake_pytensor):
    """alpha[g] + X @ beta as from_pymc lowers it (one term per column, unchanged), then fused."""
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
    assert len(m.likelihoods[0].terms) == 1 + K
    f = ir.fuse_design_columns(m)
    assert len(f.likelihoods[0].terms) == 2 and np.array_equal(f.likelihoods[0].terms[1].coef, X)
    _oracle_same(f, m, _points(m, 4, 3))


def test_lowered_tables_of_a_design_term_and_a_fused_run_are_identical():
    m = design_model("negative_binomial_log", 40, 6, group=3)
    a, b = ir.lower(m), ir.lower(ir.fuse_design_columns(as_columns(m)))
    assert np.array_equal(a.vars, b.vars) and np.array_equal(a.var_bounds, b.var_bounds)
    assert a.priors == b.priors and a.ar1 == b.ar1
    for La, Lb in zip(a.liks, b.liks):
        assert La.keys() == Lb.keys()
        for k in La:
            if k != "terms":
                assert (La[k] is None and Lb[k] is None) or np.array_equal(La[k], Lb[k]), k
        assert len(La["terms"]) == len(Lb["terms"]) == 3
        for Ta, Tb in zip(La["terms"], Lb["terms"]):
            assert Ta.keys() == Tb.keys()
            assert (Ta["coef"] is None) == (Tb["coef"] is None)
            if Ta["coef"] is not None:
                assert Ta["coef"].dtype == Tb["coef"].dtype and np.array_equal(Ta["coef"], Tb["coef"])
            assert len(Ta["factors"]) == len(Tb["factors"])
            for fa, fb in zip(Ta["factors"], Tb["factors"]):
                assert fa[:2] == fb[:2] and ((fa[2] is None) == (fb[2] is None))
            assert Ta.get("n_cols", 0) == Tb.get("n_cols", 0)
    T = a.liks[0]["terms"][1]
    assert T["n_cols"] == 6 and T["coef"].shape == (40, 6) and T["coef"].flags.c_contiguous and T["factors"][0][2] is None
    # the column form lowers as before: one table per column, no n_cols
    c = ir.lower(as_columns(m))
    assert len(c.liks[0]["terms"]) == 2 + 6 and all("n_cols" not in T for T in c.liks[0]["terms"])


def test_deterministics_and_constant_data_with_a_design_term():
    m = design_model("normal", 25, 4, group=3)
    X = m.likelihoods[0].terms[1].coef
    m.deterministics = [Deterministic("xb", 25, [Term([("beta", None)], coef=X)]),
                        Deterministic("eta", 25, [Term([("b0", None)]), Term([("beta", None)], coef=X)])]
    Q = _points(m, 6, 1).reshape(2, 3, m.n)
    post = m.constrain(Q)
    d = m.eval_deterministics(post)
    assert d["xb"].shape == (2, 3, 25)
    np.testing.assert_allclose(d["xb"], np.einsum("ik,cdk->cdi", X, post["beta"]), rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(d["eta"], post["b0"][..., None] + d["xb"], rtol=1e-14, atol=1e-14)
    cols = as_columns(m)
    cols.deterministics = [Deterministic("xb", 25, [Term([("beta", np.full(25, k, dtype=np.int32))], coef=X[:, k].copy())
                                                    for k in range(4)])]
    np.testing.assert_allclose(cols.eval_deterministics(post)["xb"], d["xb"], rtol=1e-13, atol=1e-13)
    cd = m.constant_data()
    assert np.array_equal(cd["y_coef1"], X)


def test_specialise_takes_the_design_form_of_the_logistic_glm():
    rng = np.random.default_rng(7)
    N, K = 90, 6
    X = rng.standard_normal((N, K))
    y = (rng.random(N) < 0.5).astype(np.float64)
    pri = [Prior("normal", "beta", (0.0, 1.0))]
    cols = ModelIR(vars=[Var("beta", "beta", K)], priors=pri, likelihoods=[Likelihood(
        "bernoulli_logit", y, [Term([("beta", np.full(N, k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(K)])])
    design = ModelIR(vars=[Var("beta", "beta", K)], priors=pri,
                     likelihoods=[Likelihood("bernoulli_logit", y, [Term([("beta", None)], coef=X)])])
    a, b = ir.specialise(cols, extended=True), ir.specialise(design, extended=True)
    assert a is not None and b is not None and a.name == b.name == "logistic"
    assert a.n == b.n and a.meta["n_rows"] == b.meta["n_rows"]
    assert a.data.keys() == b.data.keys() and all(np.array_equal(a.data[k], b.data[k]) for k in a.data)
    assert ir.specialise(design) is None  # only with extended=True, as for the column form
    assert ir.specialise(ir.fuse_design_columns(cols), extended=True) is not None


# ------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------
KS = [1, 2, 31, 32, 33, 200, 300, 1000, 4000]
NS = [1, 50, 1200]


def _sweep():
    """Every family meets every K; K and N vary together so that each family and each K meets every N."""
    return [(dist, K, NS[(a + b) % 3]) for a, dist in enumerate(FAMILIES) for b, K in enumerate(KS)]


def _check_device(cm, m, Q, what):
    """Both team shapes, each repeated bit for bit, against the design oracle; returns {team: (lp, g)}."""
    f = design_logp(m)
    out = logp_at_both_team_shapes(cm, Q)
    for team, (lp, g) in out.items():
        for k, q in enumerate(Q):
            lo, go = f(q)
            S = pieces_scale(m, q, lo)
            assert abs(lp[k] - lo) <= LP_TOL * S, (what, team, k, abs(lp[k] - lo) / S)
            err = np.max(np.abs(g[k] - go)) / max(1.0, np.max(np.abs(go)))
            assert err <= GRAD_TOL, (what, team, k, err)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dist", FAMILIES)
def test_device_design_term_matches_the_oracle(dist):
    from pymc_b200 import engine

    for d, K, N in _sweep():
        if d != dist:
            continue
        m = design_model(dist, N, K, seed=K + N)
        cm = engine.CompiledModel(m)
        assert cm.spec.name == "ir"
        _check_device(cm, m, _points(m, 3, K), (dist, K, N))


SHAPES = {
    "group": lambda K: design_model("poisson_log", 300, K, seed=1, group=7),
    "two_likelihoods": lambda K: two_likelihoods_model(K),
    "log_beta": lambda K: design_model("gamma_log", 120, K, seed=2, log_beta=True),
    "three_terms": lambda K: two_design_terms_model(K),
}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("K", [33, 300])
def test_device_design_term_in_composite_models(shape, K):
    from pymc_b200 import engine

    m = SHAPES[shape](K)
    Q = _points(m, 3, 9, spread=0.3)
    out = _check_device(engine.CompiledModel(m), m, Q, (shape, K))
    # the column form on the generic function, as written, agrees
    lc, gc = engine.CompiledModel(as_columns(m), specialise=False).logp_dlogp(Q)
    lp, g = out["warp"]
    assert np.all(np.abs(lp - lc) <= LP_TOL * np.array([pieces_scale(m, q, l) for q, l in zip(Q, lp)]))
    assert np.all(np.max(np.abs(g - gc), axis=1) <= GRAD_TOL * np.maximum(1.0, np.max(np.abs(gc), axis=1)))


@pytest.mark.gpu
def test_a_chain_does_not_depend_on_the_batch():
    from pymc_b200 import engine

    for m in [design_model("bernoulli_logit", 200, 45, group=5), design_model("normal", 1200, 300)]:
        cm = engine.CompiledModel(m)
        Q = _points(m, 9, 4)
        lp, g = cm.logp_dlogp(Q)
        for sl in (slice(0, 1), slice(3, 5), slice(8, 9)):
            l1, g1 = cm.logp_dlogp(Q[sl])
            assert np.array_equal(l1, lp[sl]) and np.array_equal(g1, g[sl]), (m.name, sl)


@pytest.mark.gpu
@pytest.mark.parametrize("builder", [ir.varying_intercept_logistic_ir, ir.negative_binomial_ir, ir.gamma_regression_ir,
                                     lambda: ir.gamma_regression_ir(n_obs=1200, n_features=300)])
def test_fused_and_as_written_agree_on_the_device(builder):
    from pymc_b200 import engine

    m = builder()
    Q = _points(m, 4, 11, spread=0.3)
    lf, gf = engine.CompiledModel(m).logp_dlogp(Q)
    lw, gw = engine.CompiledModel(m, specialise=False).logp_dlogp(Q)
    S = np.array([pieces_scale(m, q, l) for q, l in zip(Q, lw)])
    assert np.all(np.abs(lf - lw) <= LP_TOL * S)
    assert np.all(np.max(np.abs(gf - gw), axis=1) <= GRAD_TOL * np.maximum(1.0, np.max(np.abs(gw), axis=1)))


@pytest.mark.gpu
@pytest.mark.parametrize("team", ["warp", "cta"])
@pytest.mark.parametrize("shape,eps", [("glm", 0.15), ("group", 0.05), ("two_likelihoods", 0.1)])
def test_fixed_step_nuts_matches_the_oracle_sampler(shape, eps, team, monkeypatch):
    if team == "cta":
        monkeypatch.setenv("B200_FORCE_TEAM", "1")
    m = design_model("bernoulli_logit", 200, 40, seed=5) if shape == "glm" else SHAPES[shape](33)
    fixed_step_against_oracle(m, design_logp(m), eps, specialise=True, C=2, T=10)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle():
    m = design_model("negative_binomial_log", 150, 20, seed=6, group=4)
    fixed_step_against_oracle(m, design_logp(m), 0.2, specialise=True, dense_cov=random_dense_cov(m.n, 3, 0.05, 0.05, 5), C=2,
                              T=10)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [3, 33, 300])
def test_pointwise_log_likelihood_matches_scipy(K):
    from pymc_b200 import engine

    for m in [two_likelihoods_model(K), design_model("binomial_logit", 70, K, group=3),
              design_model("negative_binomial_log", 70, K)]:
        cm = engine.CompiledModel(m)
        Q = _points(m, 3, 8, spread=0.3)
        for lik, L in enumerate(m.likelihoods):
            ll = cm.pointwise_loglik(Q, lik=lik)
            assert ll.shape == (3, len(L.y))
            for k, q in enumerate(Q):
                x, _ = _constrained(m, q)
                want = scipy_loglik(L.dist, np.asarray(L.y), eta_of(m, L, x), lik_param(m, L, x), L.nu)
                np.testing.assert_allclose(ll[k], want, rtol=1e-12, atol=1e-12, err_msg=f"{m.name} likelihood {lik}")


def test_model_create_refuses_malformed_design_tables_through_the_c_abi():
    m = design_model("normal", 30, 8, group=3)

    def design_term(edit):
        def f(low):
            T = low.liks[0]["terms"][1]
            assert T["n_cols"] == 8
            edit(T)
        return f

    def nan(T):
        T["coef"] = T["coef"].copy()
        T["coef"][4, 5] = np.nan

    for edit, msg in [
        (lambda T: T.update(n_cols=7), r"X must have shape \(N, size of the variable\)"),
        (lambda T: T.update(factors=[(T["factors"][0][0], 8, np.zeros(30, dtype=np.int32))]), "a design term's factor takes no index"),
        (lambda T: T.update(factors=T["factors"] + [(0, 1, None)]), "a design term has exactly one factor"),
        (lambda T: T.update(factors=[]), "a design term has exactly one factor"),
        (nan, "X must be finite"),
    ]:
        err = refusal_after_edit(lambda: m, design_term(edit))
        assert err is not None and re.search(msg, err), (msg, err)
