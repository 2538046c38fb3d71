"""Zero-inflated and hurdle likelihoods of the model IR (``ir.ZI_LIKS``), with psi a constant, a scalar variable or the
logit of a linear predictor.

``_mp_lik`` writes log p(y | eta, psi) of one observation with mpmath at 40 digits from the published definitions
(pymc/distributions/mixture.py: mixture_logprob, :470-494, a logsumexp over [DiracDelta(0), f]; marginal_hurdle_logprob,
:847-870, whose count component is Truncated(f, lower=1), :826-829), with f the family's pmf / pdf and 1 - f(0) formed
without cancellation.  It is checked against scipy.stats compositions (1 - psi) [y = 0] + psi pmf(y) and
(1 - psi) [y = 0] + psi pmf(y) / (1 - pmf(0)) [y > 0].  ``_mp_logp`` is the joint log-density of a catalogue model;
S = sum |additive pieces|, and logp is compared to 1e-13 S as in tests/test_ir_closed_set.py.  A psi variable enters the
reference at its constrained double value: its accuracy is that of the constrained value, as for every variable.

CPU: the reference against scipy, the oracle (oracle/ir_numpy_zero_inflated.py) against it on the catalogue and against
central differences, the support rule, the lowered tables.  GPU: the generic device function against both, fixed-step,
lock-step and adaptive NUTS against the oracle sampler, the pointwise log-likelihood and the C ABI's refusals."""
import zlib
from functools import lru_cache

import numpy as np
import pytest
from mpmath import mp, mpf
from scipy import special, stats
from b200_helpers import (adaptive_against_oracle, fd_grad, fixed_step_against_oracle, logp_at_both_team_shapes, random_dense_cov,
                          refusal_after_edit)
from test_ir_closed_set import LP_TOL, MP_DPS

from pymc_b200 import ir
from pymc_b200.ir import Likelihood, Linear, ModelIR, Prior, Ref, Term, Var


def oracle(m):
    from oracle import ir_numpy_zero_inflated

    return ir_numpy_zero_inflated.make_logp(m)


# ------------------------------------------------------------------------------------------------------------------------
# the high-precision reference
# ------------------------------------------------------------------------------------------------------------------------
def _mp_logf(fam, y, eta, n, a):
    """log f(y) of the family at eta (mpf arguments, y an int) as its list of additive pieces."""
    if fam == "poisson_log" or (fam == "negative_binomial_log" and a > ir.NEGBIN_POISSON_ALPHA):
        return [y * eta, -mp.exp(eta), -mp.loggamma(y + 1)]
    if fam == "binomial_logit":  # log p = -log1p(e^-eta), log(1 - p) = -log1p(e^eta)
        return [mp.loggamma(n + 1), -mp.loggamma(y + 1), -mp.loggamma(n - y + 1), -y * mp.log1p(mp.exp(-eta)),
                -(n - y) * mp.log1p(mp.exp(eta))]
    if fam == "negative_binomial_log":  # n = a, p = a / (mu + a)
        mu = mp.exp(eta)
        return [mp.loggamma(y + a), -mp.loggamma(a), -mp.loggamma(y + 1), -a * mp.log1p(mu / a), y * (eta - mp.log(mu + a))]
    # Gamma, beta = a / mu
    return [a * mp.log(a), -a * eta, -mp.loggamma(a), (a - 1) * mp.log(y), -a * y * mp.exp(-eta)]


def _mp_log1m_p0(fam, eta, n, a):
    """log(1 - f(0)), formed as log(-expm1(log f(0)))."""
    if fam == "poisson_log" or a > ir.NEGBIN_POISSON_ALPHA:
        return mp.log(-mp.expm1(-mp.exp(eta)))
    return mp.log(-mp.expm1(-a * mp.log1p(mp.exp(eta) / a)))


def _mp_pieces(dist, y, eta, n, a, lpsi, l1psi):
    """log p(y | eta, psi) of one observation as its list of additive pieces."""
    fam = ir.ZI_FAMILY[dist]
    if dist.startswith("hurdle"):
        if y == 0:
            return [l1psi]
        out = [lpsi] + _mp_logf(fam, y, eta, n, a)
        return out if fam == "gamma_log" else out + [-_mp_log1m_p0(fam, eta, n, a)]
    if y == 0:
        return [mp.log(mp.exp(l1psi) + mp.exp(lpsi + mp.fsum(_mp_logf(fam, 0, eta, n, a))))]
    return [lpsi] + _mp_logf(fam, y, eta, n, a)


def _mp_lik(dist, y, eta, n, a, lpsi, l1psi):
    return mp.fsum(_mp_pieces(dist, y, eta, n, a, lpsi, l1psi))


def _mp_sigmoid_logs(z):
    """(log psi, log(1 - psi)) of psi = sigmoid(z)."""
    return -mp.log1p(mp.exp(-z)), -mp.log1p(mp.exp(z))


def _mp_constrain(m, q, exact=False):
    x, jac, o = {}, [], 0
    for v in m.vars:
        qv = [mpf(float(t)) for t in q[o : o + v.size]]
        if v.transform == "log":
            x[v.name] = [mp.exp(t) for t in qv]
            jac += qv
        elif v.transform == "interval" and exact:
            lo, hi = v.bounds
            x[v.name] = [lo + (hi - lo) / (1 + mp.exp(-t)) for t in qv]
            jac += [mp.log(hi - lo) - mp.log1p(mp.exp(-t)) - mp.log1p(mp.exp(t)) for t in qv]
        elif v.transform == "interval":  # the constrained double value; the Jacobian at 40 digits
            lo, hi = v.bounds
            z = np.asarray(q[o : o + v.size], dtype=np.float64)
            e = np.exp(-np.abs(z))
            s = np.where(z >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
            x[v.name] = [mpf(float(t)) for t in lo + (hi - lo) * s]
            jac += [mp.log(hi - lo) - mp.log1p(mp.exp(-t)) - mp.log1p(mp.exp(t)) for t in qv]
        else:
            x[v.name] = qv
        o += v.size
    return x, jac


def _mp_logp(m, q, exact=False):
    """(logp, S) of a catalogue model: normal / halfnormal priors with constant parameters, one zero-inflated or hurdle
    likelihood.  exact: an interval variable at its 40-digit constrained value (for differences in q near psi = 1, where
    the double value of 1 - psi holds only a few digits)."""
    from test_ir_bounded import _mp_eta

    with mp.workdps(MP_DPS):
        x, pieces = _mp_constrain(m, q, exact)
        for p in m.priors:
            xs = x[m.var(p.var).name]
            if p.dist == "normal":
                mu, sd = (mpf(float(t)) for t in p.params)
                pieces += [t for xi in xs for t in (-((xi - mu) / sd) ** 2 / 2, -mp.log(sd), -mp.log(2 * mp.pi) / 2)]
            else:
                assert p.dist == "halfnormal"
                sd = mpf(float(p.params[0]))
                pieces += [t for xi in xs for t in (-(xi / sd) ** 2 / 2, -mp.log(sd), mp.log(2 / mp.pi) / 2)]
        for L in m.likelihoods:
            N = len(L.y)
            eta = _mp_eta(m, L, x)
            fam = ir.ZI_FAMILY[L.dist]
            n = [mpf(float(t)) for t in np.broadcast_to(L.trials, (N,))] if fam == "binomial_logit" else [None] * N
            a = None
            if L.alpha is not None:
                a = x[m.var(L.alpha.var).name][0] if isinstance(L.alpha, Ref) else mpf(float(L.alpha))
            if isinstance(L.psi, Linear):
                zeta = _mp_eta(m, Likelihood(L.dist, L.y, L.psi.terms), x)
                logs = [_mp_sigmoid_logs(z) for z in zeta]
            else:
                p = x[m.var(L.psi.var).name][0] if isinstance(L.psi, Ref) else mpf(float(L.psi))
                logs = [(mp.log(p), mp.log1p(-p))] * N
            for i in range(N):
                yi = float(L.y[i])
                yi = int(yi) if fam != "gamma_log" else mpf(yi)
                pieces += _mp_pieces(L.dist, yi, eta[i], n[i], a, *logs[i])
        return float(mp.fsum(pieces)), float(mp.fsum(abs(t) for t in pieces))


# ------------------------------------------------------------------------------------------------------------------------
# the case catalogue
# ------------------------------------------------------------------------------------------------------------------------
def _case(dist, psi, rng, N=16, y=None, eta_off=None, zeta_off=None, alpha="var", trials=None, design=False, z0=None):
    """One likelihood: eta_i = b0 + eta_off_i (+ X beta); psi "const" (0.7), "var" (interval(0, 1), Normal(0.5, 1) prior,
    initial z0) or "logit" (g0 + zeta_off_i (+ Z gamma)); alpha "var" (log, HalfNormal(2)) or a constant."""
    fam = ir.ZI_FAMILY[dist]
    vars_ = [Var("b0", "b0", 1, initial=0.3)]
    priors = [Prior("normal", "b0", (0.0, 2.0))]
    terms = [Term([("b0", None)])]
    if eta_off is not None:
        terms.append(Term([], coef=np.asarray(eta_off, dtype=np.float64)))
    if design:
        vars_.append(Var("beta", "beta", 2))
        priors.append(Prior("normal", "beta", (0.0, 1.0)))
        terms.append(Term([("beta", None)], coef=rng.standard_normal((N, 2)) * 0.5))
    if y is None:
        y = {"poisson_log": lambda: rng.poisson(2.0, N), "negative_binomial_log": lambda: rng.poisson(3.0, N),
             "binomial_logit": lambda: rng.binomial(np.asarray(trials, dtype=int), 0.4),
             "gamma_log": lambda: rng.gamma(2.0, 1.0, N)}[fam]().astype(np.float64)
        y[rng.random(N) < 0.35] = 0.0
    kw = {}
    if fam == "binomial_logit":
        kw["trials"] = trials
    if fam in ir.DISPERSION_LIKS:
        if alpha == "var":
            vars_.append(Var("alpha_log__", "alpha", 1, "log", initial=0.5))
            priors.append(Prior("halfnormal", "alpha_log__", (2.0,)))
            kw["alpha"] = Ref("alpha_log__")
        else:
            kw["alpha"] = float(alpha)
    if psi == "const":
        p = 0.7
    elif psi == "var":
        vars_.append(Var("psi_logodds__", "psi", 1, "interval", bounds=(0.0, 1.0), initial=0.4 if z0 is None else z0))
        priors.append(Prior("normal", "psi_logodds__", (0.5, 1.0)))
        p = Ref("psi_logodds__")
    else:
        vars_.append(Var("g0", "g0", 1, initial=0.2))
        priors.append(Prior("normal", "g0", (0.0, 1.5)))
        pt = [Term([("g0", None)])]
        if zeta_off is not None:
            pt.append(Term([], coef=np.asarray(zeta_off, dtype=np.float64)))
        if design:
            vars_.append(Var("gamma", "gamma", 2))
            priors.append(Prior("normal", "gamma", (0.0, 1.0)))
            pt.append(Term([("gamma", None)], coef=rng.standard_normal((N, 2)) * 0.5))
        p = Linear(pt)
    return ModelIR(vars=vars_, priors=priors, likelihoods=[Likelihood(dist, np.asarray(y, dtype=np.float64), terms, psi=p, **kw)])


def _trials(rng, N=16):
    t = rng.integers(0, 9, N).astype(np.float64)
    t[:3] = 0.0  # n = 0: only y = 0 is possible
    return t


def _counts_1e4(rng, N=16):
    y = np.round(np.exp(rng.uniform(0.0, np.log(1e4), N)))
    y[:4] = 0.0
    return y


CASES = {}
for _d in ir.ZI_LIKS:
    _fam = ir.ZI_FAMILY[_d]
    for _p in ("const", "var", "logit"):
        CASES[f"{_d}-{_p}"] = (lambda rng, d=_d, p=_p, f=_fam: _case(d, p, rng, trials=_trials(rng) if f == "binomial_logit" else None))
    _tr = (lambda rng: _trials(rng)) if _fam == "binomial_logit" else (lambda rng: None)
    CASES[f"{_d}-design"] = (lambda rng, d=_d, tr=_tr: _case(d, "logit", rng, trials=tr(rng), design=True))
    CASES[f"{_d}-all-zero"] = (lambda rng, d=_d, tr=_tr: _case(d, "logit", rng, y=np.zeros(16), trials=tr(rng)))
    if _fam != "binomial_logit":
        _pos = (lambda rng: rng.gamma(2.0, 1.0, 16)) if _fam == "gamma_log" else (lambda rng: rng.integers(1, 6, 16).astype(float))
        CASES[f"{_d}-no-zero"] = (lambda rng, d=_d, pos=_pos: _case(d, "var", rng, y=pos(rng)))
    # eta from -700 to +30 (hurdle: y = 1 at mu ~ 1e-300), zeta = +-35
    _eta = np.array([-700.0, -690.0, -300.0, -40.0, -5.0, -1.0, 0.0, 0.5, 2.0, 5.0, 12.0, 30.0] * 2)
    _y = np.array([1, 0, 1, 0, 2, 0, 1, 3, 0, 5, 0, 1] * 2, dtype=np.float64)
    _zeta = np.array([35.0, -35.0, 0.0, 20.0, -20.0, 1.0] * 4)
    if _fam == "binomial_logit":
        _yt = np.where(_y > 0, _y, 0.0)
        CASES[f"{_d}-extreme-eta"] = (lambda rng, d=_d, yt=_yt, e=_eta, z=_zeta: _case(d, "logit", rng, N=24, y=yt, eta_off=e,
                                                                                        zeta_off=z, trials=yt + 4.0))
    elif _fam != "gamma_log":
        CASES[f"{_d}-extreme-eta"] = (lambda rng, d=_d, y=_y, e=_eta, z=_zeta: _case(d, "logit", rng, N=24, y=y, eta_off=e,
                                                                                       zeta_off=z, alpha=2.0))
    else:
        _eg = np.clip(_eta, -40.0, 30.0)
        CASES[f"{_d}-extreme-eta"] = (lambda rng, d=_d, e=_eg, z=_zeta: _case(d, "logit", rng, N=24, eta_off=e, zeta_off=z))
    for _z in (-20.0, 20.0):
        CASES[f"{_d}-psi-z{int(_z)}"] = (lambda rng, d=_d, z=_z, tr=_tr: _case(d, "var", rng, z0=z, trials=tr(rng)))
for _d in ("zero_inflated_poisson", "hurdle_poisson", "zero_inflated_negative_binomial", "hurdle_negative_binomial"):
    CASES[f"{_d}-counts-1e4"] = (lambda rng, d=_d: _case(d, "const", rng, y=_counts_1e4(rng), eta_off=np.full(16, 7.0)))
for _d in ("zero_inflated_negative_binomial", "hurdle_negative_binomial", "hurdle_gamma"):
    for _a in (1e-3, 0.5, 30.0, 1e9) + ((2e10,) if _d != "hurdle_gamma" else ()):
        CASES[f"{_d}-alpha{_a:g}"] = (lambda rng, d=_d, a=_a: _case(d, "var", rng, alpha=a))
CASE_IDS = list(CASES)


def build(cid):
    return CASES[cid](np.random.default_rng(zlib.crc32(cid.encode())))


def points(m, cid):
    rng = np.random.default_rng(zlib.crc32(cid.encode()) + 1)
    return np.array([m.initial_point() + rng.uniform(-0.5, 0.5, m.n) for _ in range(3)])


@lru_cache(maxsize=None)
def mp_reference(cid):
    m = build(cid)
    Q = points(m, cid)
    lp, S = np.array([_mp_logp(m, q) for q in Q]).T
    return Q, lp, S


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference and the oracle
# ------------------------------------------------------------------------------------------------------------------------
def _scipy_family(fam, y, eta, n=None, a=None):
    mu = np.exp(eta)
    if fam == "poisson_log":
        return stats.poisson(mu)
    if fam == "binomial_logit":
        return stats.binom(n, special.expit(eta))
    if fam == "negative_binomial_log":
        return stats.nbinom(a, a / (mu + a))
    return stats.gamma(a, scale=mu / a)


@pytest.mark.parametrize("dist", ir.ZI_LIKS)
def test_mp_reference_equals_scipy_compositions(dist):
    fam = ir.ZI_FAMILY[dist]
    rng = np.random.default_rng(zlib.crc32(dist.encode()))
    with mp.workdps(MP_DPS):
        for eta in (-2.0, -0.3, 0.4, 1.5, 3.0):
            for psi in (0.05, 0.5, 0.93):
                n, a = 7, 2.7
                f = _scipy_family(fam, None, eta, n, a)
                ys = rng.gamma(2.0, 1.5, 5) if fam == "gamma_log" else np.arange(0, 8)
                ys = np.concatenate([[0.0], ys])
                for y in ys:
                    dens = f.pdf(y) if fam == "gamma_log" else f.pmf(y)
                    if dist.startswith("hurdle"):
                        want = (1 - psi) if y == 0 else psi * dens / (1.0 if fam == "gamma_log" else 1.0 - f.pmf(0))
                    else:
                        want = (1 - psi) * (y == 0) + psi * dens
                    yy = mpf(float(y)) if fam == "gamma_log" else int(y)
                    got = _mp_lik(dist, yy, mpf(eta), mpf(n), mpf(a), mp.log(mpf(psi)), mp.log1p(-mpf(psi)))
                    assert abs(float(got) - np.log(want)) <= 1e-12 * max(1.0, abs(np.log(want))), (dist, eta, psi, y)


def test_the_catalogue_covers_every_form():
    ms = {cid: build(cid) for cid in CASE_IDS}
    kinds = {(m.likelihoods[0].dist, type(m.likelihoods[0].psi).__name__) for m in ms.values()}
    assert kinds >= {(d, k) for d in ir.ZI_LIKS for k in ("float", "Ref", "Linear")}
    ys = [np.asarray(m.likelihoods[0].y) for m in ms.values()]
    assert any(np.all(y == 0) for y in ys) and any(np.all(y > 0) for y in ys) and max(np.max(y) for y in ys) >= 5e3
    alphas = {m.likelihoods[0].alpha for m in ms.values() if isinstance(m.likelihoods[0].alpha, float)}
    assert min(alphas) <= 1e-3 and 1e9 in alphas and max(alphas) > ir.NEGBIN_POISSON_ALPHA
    assert any(np.any(np.asarray(m.likelihoods[0].trials) == 0) for m in ms.values() if m.likelihoods[0].trials is not None)
    assert any(ir.is_design(t) for m in ms.values() for t in m.likelihoods[0].terms) and \
        any(ir.is_design(t) for m in ms.values() if isinstance(m.likelihoods[0].psi, Linear) for t in m.likelihoods[0].psi.terms)


@pytest.mark.parametrize("cid", CASE_IDS)
def test_oracle_matches_the_mp_reference_and_central_differences(cid):
    m = build(cid)
    f = oracle(m)
    Q, lp_mp, S = mp_reference(cid)
    for q, want, s in zip(Q, lp_mp, S):
        lp, g = f(q)
        assert np.isfinite(lp) and np.all(np.isfinite(g)), cid
        assert abs(lp - want) <= LP_TOL * s, (cid, lp, want)
        # psi = 1 - 2e-9 at z = 20: differences of the double psi are rounding; take them of the 40-digit one
        fd = fd_grad(lambda t: _mp_logp(m, t, exact=True), q) if "psi-z20" in cid else fd_grad(f, q)
        np.testing.assert_allclose(g, fd, rtol=2e-5, atol=2e-5 * max(1.0, np.max(np.abs(g))), err_msg=cid)


def test_hurdle_density_at_tiny_mu_is_log_psi():
    """eta = -700, y = 1: log psi + log f(1) - log(1 - P0) = log psi + O(mu), finite, for the Poisson and the
    NegativeBinomial; and below mu = 1e-304 the log m form keeps it finite."""
    from oracle.ir_numpy_zero_inflated import zi_terms

    for dist, a in (("hurdle_poisson", None), ("hurdle_negative_binomial", 3.0)):
        for eta in (-700.0, -745.0, -800.0):
            lp, r, _, _, _ = zi_terms(dist, np.array([1.0]), np.array([eta]), None, a, np.log(0.3), np.log(0.7), 0.3)
            assert np.isfinite(lp[0]) and np.isfinite(r[0])
            assert abs(lp[0] - np.log(0.3)) <= 1e-12, (dist, eta, lp)


def _zi(dist="zero_inflated_poisson", y=(0, 1, 3), psi=0.6, tr=None, bounds=(0.0, 1.0), size=1, **kw):
    vars_ = [Var("b", "b", 1)]
    priors = [Prior("normal", "b", (0.0, 1.0))]
    if isinstance(psi, Ref):
        vars_.append(Var("p_x__", "p", size, tr, bounds=bounds if tr == "interval" else None))
    return ModelIR(vars=vars_, priors=priors,
                   likelihoods=[Likelihood(dist, np.asarray(y, dtype=float), [Term([("b", None)])], psi=psi, **kw)])


REFUSALS = [
    ("psi = 1", dict(psi=1.0), ir.PSI_ONE),
    ("psi = 0", dict(psi=0.0), ir.PSI_CONST),
    ("psi > 1", dict(psi=1.5), ir.PSI_CONST),
    ("psi nan", dict(psi=np.nan), ir.PSI_CONST),
    ("per-observation constant psi", dict(psi=np.array([0.5, 0.5, 0.5])), ir.PSI_BLOCK),
    ("empty logit block", dict(psi=Linear([])), ir.PSI_BLOCK),
    ("psi variable on the real line", dict(psi=Ref("p_x__")), ir.PSI_VAR),
    ("psi variable on a log transform", dict(psi=Ref("p_x__"), tr="log"), ir.PSI_VAR),
    ("psi variable on interval(0, 2)", dict(psi=Ref("p_x__"), tr="interval", bounds=(0.0, 2.0)), ir.PSI_VAR),
    ("vector psi variable", dict(psi=Ref("p_x__"), tr="interval", size=3), ir.PSI_VAR),
    ("missing psi", dict(psi=None), "needs psi"),
    ("negative count", dict(y=(-1, 0)), ir.ZI_Y),
    ("fractional count", dict(y=(0.5, 1)), ir.ZI_Y),
    ("sigma on a poisson", dict(sigma=1.0), ir.ZIP_SLOT),
    ("zib y > n", dict(dist="zero_inflated_binomial", y=(0, 4), trials=3.0), ir.ZIB_Y),
    ("zib fractional trials", dict(dist="zero_inflated_binomial", trials=2.5), "trials must be integers >= 0"),
    ("zib without trials", dict(dist="zero_inflated_binomial"), "trials must be a constant"),
    ("zinb negative count", dict(dist="zero_inflated_negative_binomial", y=(-2, 0), alpha=1.0), ir.ZI_Y),
    ("hnb without alpha", dict(dist="hurdle_negative_binomial"), "needs alpha"),
    ("hnb alpha <= 0", dict(dist="hurdle_negative_binomial", alpha=-1.0), "must be a finite constant > 0"),
    ("hurdle_gamma negative y", dict(dist="hurdle_gamma", y=(-1.0, 2.0), alpha=1.0), ir.HG_Y),
    ("hurdle_gamma infinite y", dict(dist="hurdle_gamma", y=(np.inf, 2.0), alpha=1.0), ir.HG_Y),
]


def _escape(msg):
    return msg.replace("(", r"\(").replace(")", r"\)").replace("[", r"\[").replace("]", r"\]").replace("+", r"\+")


@pytest.mark.parametrize("what,kw,msg", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_validate_refuses_each_clause(what, kw, msg):
    with pytest.raises(ValueError, match=_escape(msg)):
        _zi(**kw).validate()


def test_validate_accepts_the_allowed_forms_and_refuses_misplaced_psi():
    _zi().validate()
    _zi(psi=Ref("p_x__"), tr="interval").validate()
    _zi(psi=Ref("p_x__"), tr="interval", bounds=(0.1, 0.9)).validate()
    _zi(psi=Linear([Term([("b", None)]), Term([], coef=np.array([1.0, -2.0, 0.5]))])).validate()
    _zi(dist="zero_inflated_binomial", y=(0, 0, 2), trials=np.array([0.0, 3.0, 2.0])).validate()
    _zi(dist="hurdle_gamma", y=(0.0, 0.2, 5.0), alpha=2.0).validate()
    for d in ir.ZI_LIKS:
        for p in ("const", "var", "logit"):
            ir.zero_inflated_ir(d, p).validate()
    bad = ModelIR(vars=[Var("b", "b", 1)], priors=[Prior("normal", "b", (0.0, 1.0))],
                  likelihoods=[Likelihood("poisson_log", np.zeros(3), [Term([("b", None)])], psi=0.5)])
    with pytest.raises(ValueError, match="psi belongs to"):
        bad.validate()
    with pytest.raises(ValueError):
        ir.zero_inflated_ir("zero_inflated_gamma")


def test_lowered_tables_hold_the_psi_block_and_the_constants():
    from pymc_b200 import _lib

    m = ir.zero_inflated_ir("zero_inflated_poisson", "logit")
    low = ir.lower(m)
    L = low.liks[0]
    assert L["dist"] == ir.LIK_DISTS["zero_inflated_poisson"] == 12 and L["nu"] == 2.0 and len(L["psi"]) == 2
    off = m.offsets()
    assert L["psi"][0]["factors"] == [(off["g0"], 1, None)] and L["psi"][1]["n_cols"] == 2
    assert L["sigma_kind"] == ir.SIGMA_NONE and len(L["terms"]) == 3
    c_ir, keep = _lib.build_ir(low)  # the ctypes table holds the psi block one past the predictor's terms
    lik = _lib.IrLik.from_address(c_ir.liks)
    assert lik.n_terms == 3 and lik.nu == 2.0
    T = (_lib.IrTerm * 5).from_address(lik.terms)
    assert T[3].n_factors == 1 and T[3].f[0].offset == off["g0"] and T[4].n_cols == 2
    assert {ir.LIK_DISTS[d] for d in ir.ZI_LIKS} == set(range(12, 18))
    cv = ir.lower(ir.zero_inflated_ir("hurdle_negative_binomial", "var")).liks[0]
    mv = ir.zero_inflated_ir("hurdle_negative_binomial", "var")
    assert cv["nu"] == 0.0 and cv["psi"] == [dict(coef=None, factors=[(mv.offsets()["psi_logodds__"], 1, None)])]
    assert cv["sigma_kind"] == ir.SIGMA_REF
    cc = ir.lower(ir.zero_inflated_ir("zero_inflated_binomial", "const")).liks[0]
    assert cc["nu"] == 0.0 and cc["psi"][0]["factors"] == [] and list(cc["psi"][0]["coef"]) == [0.65]
    assert cc["sigma_kind"] == ir.SIGMA_OBS
    mc = ir.zero_inflated_ir("zero_inflated_binomial", "const")
    assert float(mc.constant_data()["y_psi"]) == 0.65 and "y_trials" in mc.constant_data()
    assert "y_psi_coef1" in m.constant_data()
    for d in ir.ZI_LIKS:
        assert ir.specialise(ir.zero_inflated_ir(d, "const")) is None
    # fuse_design_columns fuses a column run inside the psi block
    Z = np.random.default_rng(0).standard_normal((20, 2))
    cols = [Term([("gamma", np.full(20, k, dtype=np.int32))], coef=Z[:, k].copy()) for k in range(2)]
    mz = ModelIR(vars=[Var("b", "b", 1), Var("gamma", "gamma", 2)], priors=[Prior("normal", "b", (0.0, 1.0)),
                                                                          Prior("normal", "gamma", (0.0, 1.0))],
                 likelihoods=[Likelihood("hurdle_poisson", np.zeros(20), [Term([("b", None)])], psi=Linear(cols))])
    fz = ir.fuse_design_columns(mz)
    assert len(fz.likelihoods[0].psi.terms) == 1 and np.array_equal(fz.likelihoods[0].psi.terms[0].coef, Z)
    q = np.array([0.1, 0.3, -0.2])
    assert abs(oracle(fz)(q)[0] - oracle(mz)(q)[0]) <= 1e-12 * abs(oracle(mz)(q)[0])


def test_constants_of_c0_match_the_oracle_split():
    """The constants prepare_ir folds (-lgamma(y + 1), binomln(n, y), lgamma(y + a) - lgamma(a), and the Gamma normaliser
    over the N+ positive y) are exactly what separates logp at two values of the predictor-free parts: checked by the
    oracle's per-observation log-likelihood, which includes them, against the mp reference on the y > 0 observations."""
    m = ir.zero_inflated_ir("hurdle_gamma", "const", n_obs=40)
    L = m.likelihoods[0]
    y = np.asarray(L.y)
    pos = y > 0
    assert 0 < pos.sum() < len(y)
    f = oracle(m)
    q = m.initial_point() + 0.1
    x, _ = f.constrained(q)
    ll = f.loglik(L, x)
    a = x[m.offsets()["alpha_log__"]]
    eta = f.eta(L, x)[0]
    want = np.where(pos, np.log(0.65) + stats.gamma.logpdf(np.where(pos, y, 1.0), a, scale=np.exp(eta) / a), np.log(0.35))
    np.testing.assert_allclose(ll, want, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: the generic device function
# ------------------------------------------------------------------------------------------------------------------------
def _device(m):
    from pymc_b200 import engine

    return engine.CompiledModel(m, specialise=False)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", CASE_IDS)
def test_device_logp_matches_the_mp_reference_and_the_oracle(cid):
    m = build(cid)
    cm = _device(m)
    f = oracle(m)
    Q, lp_mp, S = mp_reference(cid)
    lo = np.array([f(q)[0] for q in Q])
    go = np.array([f(q)[1] for q in Q])
    for team, (lp, g) in logp_at_both_team_shapes(cm, Q).items():
        assert np.all(np.abs(lp - lp_mp) <= LP_TOL * S), (cid, team, lp - lp_mp)
        assert np.all(np.abs(lp - lo) <= LP_TOL * S), (cid, team, lp - lo)
        scale = np.maximum(1.0, np.max(np.abs(go), axis=1, keepdims=True))
        err = np.max(np.abs(g - go) / scale, axis=1)
        assert np.all(err <= 1e-11), (cid, team, err)


@pytest.mark.gpu
@pytest.mark.parametrize("dist,psi", [("zero_inflated_poisson", "logit"), ("zero_inflated_negative_binomial", "var"),
                                      ("hurdle_gamma", "logit"), ("hurdle_negative_binomial", "const"),
                                      ("zero_inflated_binomial", "logit")])
def test_fixed_step_nuts_matches_the_oracle_sampler(dist, psi):
    m = ir.zero_inflated_ir(dist, psi)
    fixed_step_against_oracle(m, oracle(m), 0.05)


@pytest.mark.gpu
def test_lockstep_dense_mass_run_matches_the_oracle():
    m = ir.zero_inflated_ir("zero_inflated_negative_binomial", "logit", n_obs=120)
    fixed_step_against_oracle(m, oracle(m), 0.3, dense_cov=random_dense_cov(m.n, 2, 0.01, 0.05, 12), C=2, T=10)


@pytest.mark.gpu
def test_adaptive_run_matches_the_oracle_posterior_and_recovers_psi():
    """64 device chains against 8 oracle chains on a zero-inflated Poisson with a random psi: posterior means within 4 MCSE
    (an effective-size-free bound, SE of the mean of the pooled draws), standard deviations within 25 %; the posterior of
    psi from sample_b200_nuts holds the simulated 0.6 within three posterior standard deviations (the spread the data
    leave) plus four MCSEs (bounded with an effective size of a tenth of the draws)."""
    import pymc_b200

    m = ir.zero_inflated_ir("zero_inflated_poisson", "var", n_obs=400)
    adaptive_against_oracle(m, oracle(m), chain_seed=23, spread=0.5, philox_seed=5, oracle_seed=200, se_bound=4.0)
    res = pymc_b200.sample_b200_nuts(300, tune=300, chains=8, random_seed=3, model=m, compute_convergence_checks=False)
    psi = np.asarray(res.posterior["psi"]).ravel()
    assert np.all((psi > 0) & (psi < 1))
    assert abs(psi.mean() - 0.6) <= 3.0 * psi.std() + 4.0 * psi.std() / np.sqrt(len(psi) / 10)


@pytest.mark.gpu
def test_pointwise_log_likelihood_and_the_log_likelihood_group_match_scipy():
    import pymc_b200

    def scipy_ll(m, q):
        f = oracle(m)
        L = m.likelihoods[0]
        fam = ir.ZI_FAMILY[L.dist]
        y = np.asarray(L.y)
        out = np.empty(q.shape[:-1] + (len(y),))
        for ix in np.ndindex(*q.shape[:-1]):
            x, _ = f.constrained(q[ix])
            eta = f.eta(L, x)[0]
            lpsi, l1psi, p, _, _ = f.psi(L, x)
            psi = np.exp(lpsi)
            nt, a, _ = f.family_params(L, x)
            d = _scipy_family(fam, y, eta, nt, a)
            if fam == "gamma_log":
                dens = d.logpdf(np.where(y > 0, y, 1.0))
                out[ix] = np.where(y == 0, np.log1p(-psi), np.log(psi) + dens)
            elif L.dist.startswith("hurdle"):
                out[ix] = np.where(y == 0, np.log1p(-psi), np.log(psi) + d.logpmf(y) - np.log(d.sf(0)))
            else:
                out[ix] = np.where(y == 0, np.log((1 - psi) + psi * d.pmf(0)), np.log(psi) + d.logpmf(y))
        return out

    for d in ir.ZI_LIKS:
        for p in ("const", "var", "logit"):
            m = ir.zero_inflated_ir(d, p, n_obs=60)
            cm = _device(m)
            q = m.initial_point() + np.random.default_rng(4).uniform(-0.3, 0.3, (2, 3, m.n))
            np.testing.assert_allclose(cm.pointwise_loglik(q), scipy_ll(m, q), rtol=1e-10, atol=1e-10, err_msg=f"{d}-{p}")
    for m in (ir.zero_inflated_ir("hurdle_negative_binomial", "logit"), ir.zero_inflated_ir("zero_inflated_binomial", "var")):
        res = pymc_b200.sample_b200_nuts(20, tune=60, chains=4, random_seed=3, model=m, keep_untransformed=True,
                                         idata_kwargs={"log_likelihood": True}, compute_convergence_checks=False)
        ll = res.log_likelihood["y"]
        assert ll.shape == (4, 20, len(m.likelihoods[0].y))
        np.testing.assert_allclose(ll, scipy_ll(m, res.unconstrained), rtol=1e-10, atol=1e-10)


def test_model_create_refuses_malformed_psi_and_y_tables_through_the_c_abi():
    def set_y(low, v, i=0):
        low.liks[0]["y"] = low.liks[0]["y"].copy()
        low.liks[0]["y"][i] = v

    def set_psi(low, v):
        low.liks[0]["psi"][0]["coef"] = np.array([v])

    zip_c = lambda: ir.zero_inflated_ir("zero_inflated_poisson", "const")  # noqa: E731
    zip_v = lambda: ir.zero_inflated_ir("zero_inflated_poisson", "var")  # noqa: E731
    zi_v = lambda: _zi(psi=Ref("p_x__"), tr="interval")  # noqa: E731  (no prior on psi: the psi rule alone refuses)
    zib = lambda: ir.zero_inflated_ir("zero_inflated_binomial", "logit")  # noqa: E731
    hg = lambda: ir.zero_inflated_ir("hurdle_gamma", "const")  # noqa: E731
    hnb = lambda: ir.zero_inflated_ir("hurdle_negative_binomial", "logit")  # noqa: E731
    b0 = lambda low: ir.lower(zip_c()).liks[0]["terms"][0]["factors"][0][0]  # noqa: E731
    cases = [
        (zip_c, lambda low: set_psi(low, 1.0), ir.PSI_ONE),
        (zip_c, lambda low: set_psi(low, 0.0), ir.PSI_CONST),
        (zip_c, lambda low: set_psi(low, np.nan), ir.PSI_CONST),
        (zip_c, lambda low: set_psi(low, -0.5), ir.PSI_CONST),
        (zip_c, lambda low: low.liks[0]["psi"][0].update(coef=None), ir.PSI_BLOCK),
        (zip_c, lambda low: low.liks[0]["psi"][0].update(factors=[(b0(low), 1, None)]), ir.PSI_BLOCK),
        (zip_v, lambda low: low.liks[0]["psi"][0].update(factors=[(b0(low), 1, None)]), ir.PSI_VAR),  # b0: real line
        (zi_v, lambda low: low.var_bounds.__setitem__((1, 1), 2.0), ir.PSI_VAR),  # interval(0, 2)
        (zip_c, lambda low: low.liks[0].update(nu=-1.0), ir.PSI_NU),
        (zip_c, lambda low: low.liks[0].update(nu=0.5), ir.PSI_NU),
        (zip_c, lambda low: set_y(low, -1.0), ir.ZI_Y),
        (zip_c, lambda low: set_y(low, 1.5), ir.ZI_Y),
        (zip_c, lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_CONST, sigma_value=1.0), ir.ZIP_SLOT),
        (zib, lambda low: set_y(low, 1e3), ir.ZIB_Y),
        (zib, lambda low: low.liks[0].update(sigma_kind=ir.SIGMA_NONE), "trials must be a constant"),
        (hg, lambda low: set_y(low, -1.0), ir.HG_Y),
        (hg, lambda low: set_y(low, np.inf), ir.HG_Y),
        (hnb, lambda low: set_y(low, 2.5), ir.ZI_Y),
        (hnb, lambda low: low.liks[0].update(y_var=1), "latent factor"),
    ]
    for builder, edit, msg in cases:
        err = refusal_after_edit(builder, edit)
        assert err is not None and msg in err, (msg, err)
