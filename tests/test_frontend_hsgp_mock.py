"""CPU: ``from_pymc`` on imitation graphs (tests/test_frontend_mock.py's stand-ins) of the HSGP term
phi @ (beta * sqrt(psd)) that pm.gp.HSGP.prior (non-centred) and prior_linearized build, with psd as cov.py's
ExpQuad / Matern52 / Matern32 ``power_spectral_density`` writes it (c * prod(ls) * exp(-0.5 dot(square(omega),
square(ls))) or (num / den) * prod(ls) * power(nu + dot(...), -(D + nu) / 2), ls = ones(D) * ls), optionally times eta**2
or a constant.  Constant subgraphs stand as the constants PyTensor's constant folding makes of them.  Each accepted form
must lower to the spectral term a hand-built IR has, with the same density; the forms outside the closed set are refused
by name."""
import re
import sys

import numpy as np
import pytest
from test_frontend_mock import Constant, Dot, FakeModel, LogTransform, Subtensor, apply, bcast, elem, fake_pytensor, rv  # noqa: F401

from oracle import ir_numpy_hsgp
from pymc_b200 import ir

N = 30


def _psd(cov, omega, lsx, D):
    """cov.py's power_spectral_density graph of ExpQuad / Matern52 / Matern32 at omega, with ls = lsx (already ones(D) * ls)"""
    dot = apply(Dot(), elem("Sqr", Constant(omega)), elem("Sqr", lsx))
    c = np.exp(ir.spectral_log_const(cov, D)[0])
    head = elem("Mul", Constant(c), apply(Prod(), lsx))
    if cov == "expquad":
        return elem("Mul", head, elem("Exp", elem("Mul", Constant(-0.5), dot)))
    nu = 5.0 if cov == "matern52" else 3.0
    return elem("Mul", head, elem("Pow", elem("Add", Constant(nu), dot), Constant(-(D + nu) / 2.0)))


def _model(cov="expquad", D=1, ls="free", amp="eta2", drop_first=False, m=8, order="z_first", psd_edit=None):
    rng = np.random.default_rng(5)
    X = rng.uniform(0.0, 5.0, (N, D))
    Phi, omega, _, _ = ir.hsgp_basis(X, [m] * D, c=1.5)
    Phi_kept = Phi[:, 1:] if drop_first else Phi
    M = FakeModel("hsgp")
    lsv = None
    if ls == "free":
        lsv = M.free(rv("InvGammaRV", "ell", Constant(4.0), Constant(6.0)), D, LogTransform(), initial=np.zeros(D))
    elif ls == "iso":
        lsv = M.free(rv("InvGammaRV", "ell", Constant(4.0), Constant(6.0)), 1, LogTransform())
    eta = M.free(rv("HalfNormalRV", "eta", Constant(0.0), Constant(1.0)), 1, LogTransform()) if amp in ("eta2", "eta") else None
    z = M.free(rv("NormalRV", "f_hsgp_coeffs", Constant(0.0), Constant(1.0)), Phi_kept.shape[1])
    sigma = M.free(rv("HalfNormalRV", "sigma", Constant(0.0), Constant(1.0)), 1, LogTransform())
    if ls == "inv":
        lsi = M.free(rv("HalfNormalRV", "ell_inv", Constant(0.0), Constant(1.0)), 1, LogTransform())
        lsx = elem("Mul", Constant(np.ones(D)), bcast(elem("TrueDiv", Constant(1.0), lsi)))
    elif ls == "const":
        lsx = elem("Mul", Constant(np.ones(D)), Constant(0.9))
    else:
        lsx = elem("Mul", Constant(np.ones(D)), bcast(lsv) if ls == "iso" else lsv)
    psd = _psd(cov, omega, lsx, D)
    if amp == "eta2":
        psd = elem("Mul", elem("Pow", bcast(eta), Constant(2.0)), psd)
    elif amp == "eta":
        psd = elem("Mul", bcast(eta), psd)
    elif amp == "const":
        psd = elem("Mul", Constant(2.25), psd)
    if psd_edit is not None:
        psd = psd_edit(psd)
    if drop_first:
        psd = apply(Subtensor(), psd, Constant(1))
    sq = elem("Sqrt", psd)
    b = elem("Mul", z, sq) if order == "z_first" else elem("Mul", sq, z)
    f = apply(Dot(), Constant(Phi_kept), b)
    y = rng.normal(0.0, 1.0, N)
    M.observe(rv("NormalRV", "y", f, sigma), y)
    return M, Phi_kept, (omega[1:] if drop_first else omega), y


def _reference(cov, Phi, omega, y, ls, amp, D):
    """The same model built by hand."""
    M = Phi.shape[1]
    vars_, priors = [], []
    lsv = np.full(D, 0.9) if ls == "const" else ir.Ref("ell_log__")
    if ls in ("free", "iso"):
        vars_.append(ir.Var("ell_log__", "ell", D if ls == "free" else 1, "log"))
        priors.append(ir.Prior("inversegamma", "ell_log__", (4.0, 6.0)))
    a = 1.5 if amp == "const" else (1.0 if amp is None else ir.Ref("eta_log__"))
    if amp == "eta2":
        vars_.append(ir.Var("eta_log__", "eta", 1, "log"))
        priors.append(ir.Prior("halfnormal", "eta_log__", (1.0,)))
    vars_ += [ir.Var("f_hsgp_coeffs", "f_hsgp_coeffs", M), ir.Var("sigma_log__", "sigma", 1, "log")]
    priors += [ir.Prior("normal", "f_hsgp_coeffs", (0.0, 1.0)), ir.Prior("halfnormal", "sigma_log__", (1.0,))]
    t = ir.Term([("f_hsgp_coeffs", None)], coef=Phi, spectral=ir.Spectral(cov, omega, lsv, a))
    return ir.ModelIR(vars_, priors, [ir.Likelihood("normal", y, [t], sigma=ir.Ref("sigma_log__"))])


class Prod:
    pass


def _fold(x):
    """The value of an imitation graph made of constants only, as PyTensor's constant folding computes it; raises at
    anything that depends on a variable."""
    if isinstance(x, Constant):
        return np.asarray(x.data, dtype=np.float64)
    if x.owner is None:
        raise ValueError("not a constant")
    op, ins = x.owner.op, x.owner.inputs
    if isinstance(op, Dot):
        return np.dot(_fold(ins[0]), _fold(ins[1]))
    if isinstance(op, Prod):
        return np.prod(_fold(ins[0]))
    if type(op).__name__ == "DimShuffle":
        return _fold(ins[0])
    if isinstance(op, Subtensor):
        return _fold(ins[0])[int(_fold(ins[1])):]
    kind = type(getattr(op, "scalar_op", None)).__name__.lower()
    v = [_fold(a) for a in ins]
    fns = {"mul": lambda: np.prod(np.broadcast_arrays(*v), axis=0), "add": lambda: sum(v), "sqr": lambda: v[0] ** 2,
           "sqrt": lambda: np.sqrt(v[0]), "exp": lambda: np.exp(v[0]), "pow": lambda: v[0] ** v[1],
           "truediv": lambda: v[0] / v[1]}
    if kind not in fns:
        raise ValueError("not a constant")
    return fns[kind]()


@pytest.fixture
def folding(fake_pytensor):
    """The stand-ins with PyTensor's constant folding, which pymc.pytensorf.constant_fold gives a real graph: every
    constant subgraph (the density's constants, square(omega), a fixed ls and what it makes) has a value."""
    def constant_fold(xs, raise_not_constant=True):
        return [_fold(x) for x in xs]

    sys.modules["pymc.pytensorf"].constant_fold = constant_fold
    yield


@pytest.mark.parametrize("fold", [False, True], ids=["graph", "folded"])
@pytest.mark.parametrize("cov,D,ls,amp,drop,order", [
    ("expquad", 1, "free", "eta2", False, "z_first"),
    ("matern52", 1, "iso", "eta2", True, "psd_first"),
    ("matern32", 2, "free", "eta2", False, "z_first"),
    ("expquad", 2, "iso", "const", False, "z_first"),
    ("matern52", 2, "free", None, True, "z_first"),
    ("expquad", 1, "const", "eta2", False, "z_first"),
    ("matern32", 2, "const", "eta2", True, "psd_first"),
    ("matern52", 1, "const", "const", False, "z_first"),
])
def test_hsgp_graphs_lower_to_spectral_terms(request, fake_pytensor, fold, cov, D, ls, amp, drop, order):
    from pymc_b200 import from_pymc

    if fold:
        request.getfixturevalue("folding")
    M, Phi, omega, y = _model(cov, D, ls, amp, drop, order=order)
    m = from_pymc(M)
    t = m.likelihoods[0].terms[0]
    assert t.spectral is not None and t.spectral.cov == cov
    np.testing.assert_allclose(t.spectral.omega, omega, rtol=1e-15)
    np.testing.assert_array_equal(t.coef, Phi)
    ref = _reference(cov, Phi, omega, y, ls, amp, D)
    f, g = ir_numpy_hsgp.make_logp(m), ir_numpy_hsgp.make_logp(ref)
    rng = np.random.default_rng(1)
    off_m, off_r = m.offsets(), ref.offsets()
    for _ in range(3):
        qr = ref.initial_point() + rng.uniform(-0.5, 0.5, ref.n)
        qm = np.empty(m.n)
        for v in ref.vars:
            qm[off_m[v.name] : off_m[v.name] + v.size] = qr[off_r[v.name] : off_r[v.name] + v.size]
        (a, ga), (b, gb) = f(qm), g(qr)
        assert abs(a - b) <= 1e-12 * abs(b)
        for v in ref.vars:
            np.testing.assert_allclose(ga[off_m[v.name] : off_m[v.name] + v.size], gb[off_r[v.name] : off_r[v.name] + v.size],
                                       rtol=1e-12, atol=1e-12)


def test_inversegamma_prior_maps_to_the_ir_prior(fake_pytensor):
    from pymc_b200 import from_pymc

    M, *_ = _model()
    m = from_pymc(M)
    p = next(p for p in m.priors if p.var == "ell_log__")
    assert p.dist == "inversegamma" and p.params == (4.0, 6.0)


def _sum_of_kernels(psd):
    return elem("Add", psd, psd)


def _product_of_kernels(psd):
    return elem("Mul", psd, _psd("expquad", np.ones((8, 1)), elem("Mul", Constant(np.ones(1)), Constant(0.5)), 1))


def _bessel(psd):
    return elem("Mul", psd, elem("Ive", Constant(1.0), bcast(Constant(2.0))))


@pytest.mark.parametrize("kw,words", [
    (dict(amp="eta"), "eta * cov with a random eta"),
    (dict(ls="inv"), "ls_inv"),
    (dict(psd_edit=_sum_of_kernels), "sums of kernels"),
    (dict(psd_edit=_product_of_kernels), "products of kernels"),
    (dict(psd_edit=_bessel), "HSGPPeriodic"),
])
def test_forms_outside_the_closed_set_are_refused_by_name(fake_pytensor, kw, words):
    from pymc_b200 import from_pymc

    M, *_ = _model(**kw)
    with pytest.raises(NotImplementedError, match=re.escape(words)):
        from_pymc(M)


def test_the_centred_form_is_refused_by_name(fake_pytensor):
    from pymc_b200 import from_pymc

    # centred: beta ~ Normal(0, sqrt_psd), f = phi @ beta
    rng = np.random.default_rng(2)
    X = rng.uniform(0.0, 5.0, (N, 1))
    Phi, omega, _, _ = ir.hsgp_basis(X, [6], c=1.5)
    C = FakeModel("centred")
    ell = C.free(rv("InvGammaRV", "ell", Constant(4.0), Constant(6.0)), 1, LogTransform())
    sq = elem("Sqrt", _psd("expquad", omega, elem("Mul", Constant(np.ones(1)), bcast(ell)), 1))
    beta = C.free(rv("NormalRV", "f_hsgp_coeffs", Constant(0.0), sq), 6)
    C.observe(rv("NormalRV", "y", apply(Dot(), Constant(Phi), beta), Constant(1.0)), rng.normal(0.0, 1.0, N))
    with pytest.raises(NotImplementedError, match="centred HSGP parametrisation"):
        from_pymc(C)


def _no_prod(psd):
    """the ExpQuad density without its prod(ls) factor"""
    x = psd.owner.inputs[1]  # eta**2 * (c * prod(ls) * exp(...)): the density
    c_prod, ex = x.owner.inputs
    return elem("Mul", psd.owner.inputs[0], elem("Mul", c_prod.owner.inputs[0], ex))


def _other_prod(psd):
    """prod() of another vector in place of prod(ls)"""
    x = psd.owner.inputs[1]
    c_prod, ex = x.owner.inputs
    return elem("Mul", psd.owner.inputs[0], elem("Mul", elem("Mul", c_prod.owner.inputs[0],
                                                              apply(Prod(), Constant(np.full(1, 2.0)))), ex))


@pytest.mark.parametrize("edit", [_no_prod, _other_prod])
def test_a_density_without_prod_ls_is_refused(fake_pytensor, edit):
    from pymc_b200 import from_pymc

    M, *_ = _model("expquad", 1, "free", "eta2", psd_edit=edit)
    with pytest.raises(NotImplementedError, match=re.escape("prod(ls) of the ls in its exponent")):
        from_pymc(M)


def test_a_folded_constant_sqrt_psd_lowers_to_a_design_term(fake_pytensor):
    """phi @ (beta * s) with s already M constants (a fixed sqrt_psd): the design term Phi diag(s)."""
    from pymc_b200 import from_pymc

    rng = np.random.default_rng(4)
    Phi = rng.standard_normal((N, 6))
    s = rng.uniform(0.1, 1.0, 6)
    M = FakeModel("fixed")
    z = M.free(rv("NormalRV", "f_hsgp_coeffs", Constant(0.0), Constant(1.0)), 6)
    M.observe(rv("NormalRV", "y", apply(Dot(), Constant(Phi), elem("Mul", z, Constant(s))), Constant(1.0)),
              rng.normal(0.0, 1.0, N))
    m = from_pymc(M)
    t = m.likelihoods[0].terms[0]
    assert t.spectral is None
    np.testing.assert_array_equal(t.coef, Phi * s[None, :])
