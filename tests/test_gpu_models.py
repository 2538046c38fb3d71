"""The hand-written model kernels (csrc/models.cuh) against a high-precision reference, at every instantiation and data layout.

Kernels under test, all three through every kernel that evaluates them:
  * ``EightSchoolsModel::eval<NPL, 1>`` (chain = warp, NPL in {1, 2, 4, 6, 8}: J in {1, 30, 31, 33, 62, 63, 126, 127, 190,
    191, 254} are the NPL edges at n = J + 2, and J = 33 takes a second lane pass);
  * ``RadonModel::eval<NPL, 1>`` (chain = warp; J in {1, 13, 14, 29, 30, 61, 62, 93, 94, 125} are the NPL edges at
    n = 2 J + 5) over county layouts that drive its row padding: empty counties (county 0, county J - 1, more than 32 of them
    so a lane loops), one dominant county, all singletons, sizes = 0, 1, 2, 3 (mod 4), exactly 32 and 33 non-empty counties
    and tied sizes (the stable sort);
  * ``StochVolModel::eval<NPL, 8>`` (chain = CTA; T in {2, 509, 510, 1021, 1022, 2045, 2046, 3069, 3070, 4093} are the NPL
    edges at n = T + 3).
Each is run as ``b200_logp_dlogp`` (``SMALL = false``), batched and at a single point (bit-equal to each other), and inside the
persistent fixed-step NUTS kernel (``SMALL = true``) against oracle/nuts_numpy.Oracle: identical tree sizes, positions within
1e-9, and the ``model_logp`` of every draw bit-equal to ``logp_dlogp`` at that draw.  Two Radon layouts are large enough that
the NUTS kernel keeps one tree level (``hot = 1``) or none (``hot = 0``) in shared memory; they are picked with a replica of
``prepare_radon``'s row rule and ``nuts_warp_smem_bytes`` that a CPU test pins against a hand-worked table.

Reference.  The three densities and their analytic gradients are restated here in ``np.longdouble`` (64-bit significand on
x86-64) from ``ModelSpec.data`` alone; a CPU test checks them against a 40-digit mpmath evaluation of the models' definitions
and against central differences of that mpmath log-density.  The same model written as IR and run on the generic IR device
function (``specialise=False``) is a third comparator.

Bound.  Every output o (logp, each gradient entry) is assembled from terms t_i; S(o) is the sum of the magnitude envelopes of
those terms, where a term's envelope bounds every intermediate it is formed from (Radon: m_i = |y_i| + |alpha_c| + |beta_c x_i|
for the residual; Eight Schools: |y_j| + |mu| + tau |theta_j|; StochVol: w_t (1 + |mu| + |h_t|) for w_t = y_t^2 exp(-(mu + h_t)),
whose exp argument carries an absolute rounding error u |mu + h_t|, and |h_t| + |h_(t-1)| for the innovation; a squared
residual r^2 has envelope 2 |r| m; Radon's padding slots add 2 npad |alpha_c| to a county's residual sums).  The test asserts

    |kernel - ref| <= c u S,   u = 2^-53,   c = L + R + 20

with L the longest serial chain of additions one lane or thread performs, R the depth of the cross-lane reduction, and 20 for
forming one term and assembling the output:
  * L: Eight Schools ceil(J / 32) (a lane's elements); Radon ceil(K_row / 2) + 2 (the two interleaved per-row accumulators and
    their merge with the padding correction) + M (the rows) + ceil(E / 32) (the empty-county loop), K_row the longest padded
    row; StochVol NPL (a thread's time steps);
  * R: 5 for the warp butterfly (warp_sum_n / warp_sum_bcast_n), 12 for the chain-per-CTA team sum (5 within each warp, then
    the 8 warp partials added in series);
  * 20: at most 8 roundings in forming one term relative to its envelope (exp and log1p are within 1 ulp in CUDA's fp64
    libm; each product, fma or subtraction adds one), and at most 12 additions assembling the output from the reduced sums.
This is the first-order forward-error bound of that summation structure, so it cannot be flaky, and a dropped, duplicated or
padded term misses it by orders of magnitude.  Against the generic IR function the allowance is the sum of both bounds, with
c_ir = N + n + 20 for the generic function (N observations or time steps, n unknowns: the bound of any summation order).
Every case writes its largest err / (u S) to the parity report before it asserts.

Each case puts its largest entry at a boundary: the largest |x| in the last county, the largest a_c, b_c at county J - 1, the
largest |y_j| and theta_j at j = J - 1, the largest |y_t| and |mu + h_t| at t = T - 1.  The sampler checks run each layout with
data of unit scale: on the extreme data the first leapfrog of every trajectory diverges, which would check nothing.
"""
import math

import numpy as np
import pytest

from test_gpu_fullsize import _report

LD = np.longdouble
U = 2.0**-53
HAVE_LD = np.finfo(np.longdouble).nmant >= 63
needs_ld = pytest.mark.skipif(not HAVE_LD, reason="np.longdouble has fewer than 63 significand bits on this platform")

_WORST = {}  # kernel -> largest err / (u S) over the cases run

# ------------------------------------------------------------------------------------------------------------------------
# replicas of the host-side rules (csrc/b200nuts.cu, csrc/nuts_warp.cuh)
# ------------------------------------------------------------------------------------------------------------------------
MAX_SMEM = 227 * 1024
K_MAX_LEVELS = 12


def npl_warp(n):
    need = -(-n // 32)
    return next((o for o in (1, 2, 4, 6, 8) if need <= o), 0)


def npl_team(n):
    need = -(-n // 256)
    return next((o for o in (2, 4, 8, 12, 16) if need <= o), 0)


def radon_layout(county, J):
    """prepare_radon's rows: non-empty counties sorted by size (stable, largest first), dealt 32 to a row, each row padded
    to its longest county rounded up to 4; K = the rows' lengths + 4 (the prefetched block).  -> dict(K, M, E, rows, pad,
    shared) with pad[c] the padding slots of county c and shared the bytes RadonModel stages into shared memory."""
    sizes = np.bincount(np.asarray(county), minlength=J)
    order = sorted((c for c in range(J) if sizes[c] > 0), key=lambda c: -sizes[c])
    M = max(1, -(-len(order) // 32))
    rows, pad = [], np.zeros(J, dtype=np.int64)
    for j in range(M):
        members = order[32 * j:32 * j + 32]
        L = (max((sizes[c] for c in members), default=0) + 3) & ~3
        rows.append(L)
        for c in members:
            pad[c] = L - sizes[c]
    K = sum(rows) + 4
    shared = K * 32 * 16 + (M * 32 + ((M + 3) & ~3)) * 4
    return dict(K=K, M=M, E=int(np.sum(sizes == 0)), rows=rows, pad=pad, shared=shared)


def nuts_warp_smem_bytes(NP, hot, W):
    vecs = 2 + (3 if W > 1 else 0) + ((2 + 4 * (hot - 1)) if hot > 0 else 0)
    return vecs * NP * 8 + 5 * K_MAX_LEVELS * 8 + (W * 8 * 8 if W > 1 else 0)


def radon_hot_level(shared, n, max_td=10):
    """Tree levels the NUTS launch keeps in shared memory for a chain-per-warp model (NutsLaunch), or None when even hot = 0
    does not fit -- which b200_model_create refuses, as it refuses a logp launch that does not fit."""
    NP = 32 * npl_warp(n)
    data = (shared + 15) & ~15
    if data + 8 * 2 * NP * 8 > MAX_SMEM:
        return None
    hot = min(2, max_td)
    while data + 8 * nuts_warp_smem_bytes(NP, hot, 1) > MAX_SMEM and hot > 0:
        hot -= 1
    return hot if data + 8 * nuts_warp_smem_bytes(NP, hot, 1) <= MAX_SMEM else None


def _dominant_sizes(dominant, J=85):
    s = np.full(J, 2)
    s[-1] = dominant
    return s


def _dominant_for_hot(hot, J=85):
    """The smallest dominant county (the others hold 2 observations each) at which the NUTS launch keeps `hot` levels."""
    for d in range(2, 2000):
        s = _dominant_sizes(d, J)
        lay = radon_layout(np.repeat(np.arange(J), s), J)
        if radon_hot_level(lay["shared"], 2 * J + 5) == hot:
            return d
    raise AssertionError(hot)


# ------------------------------------------------------------------------------------------------------------------------
# reference (longdouble): logp, gradient and the envelopes S
# ------------------------------------------------------------------------------------------------------------------------
def _ld(a):
    return np.asarray(a, dtype=LD)


HALF_LOG_2PI = np.log(LD(8) * np.arctan(LD(1))) / 2


def _halfcauchy(z, x, beta):
    """HalfCauchy(beta) of x = exp(z) with the log Jacobian, its z-derivative, and both envelopes."""
    u = (x / beta) ** 2
    c = np.log(LD(2)) - np.log(LD(4) * np.arctan(LD(1))) - np.log(LD(beta))
    val = c - np.log1p(u) + z
    d = 1 - 2 * u / (1 + u)
    return val, d, abs(c) + np.log1p(u) + np.abs(z) + 1, 1 + 2 * u / (1 + u)


def eight_ref(y, sigma, Q):
    y, s, Q = _ld(y), _ld(sigma), _ld(np.atleast_2d(Q))
    J = len(y)
    mu, lt, tt = Q[:, :1], Q[:, 1:2], Q[:, 2:]
    tau = np.exp(lt)
    d = y - (mu + tau * tt)
    is2 = 1 / (s * s)
    r = d * is2
    a = np.abs(y) + np.abs(mu) + tau * np.abs(tt)
    hc, dhc, S_hc, S_dhc = _halfcauchy(lt[:, 0], tau[:, 0], 5)
    mu0 = mu[:, 0]
    log5 = np.log(LD(5))
    lp = (-mu0 * mu0 / 50 - HALF_LOG_2PI - log5) + hc - (tt * tt).sum(1) / 2 - J * HALF_LOG_2PI \
        + (-d * r / 2 - np.log(s)).sum(1) - J * HALF_LOG_2PI
    g = np.empty(Q.shape, dtype=LD)
    g[:, 0] = -mu0 / 25 + r.sum(1)
    g[:, 1] = tau[:, 0] * (r * tt).sum(1) + dhc
    g[:, 2:] = tau * r - tt
    S_lp = mu0 * mu0 / 50 + HALF_LOG_2PI + log5 + S_hc + (tt * tt).sum(1) / 2 + 2 * J * HALF_LOG_2PI \
        + (np.abs(d) * a * is2 + np.abs(np.log(s))).sum(1)
    S_g = np.empty(Q.shape, dtype=LD)
    S_g[:, 0] = np.abs(mu0) / 25 + (a * is2).sum(1)
    S_g[:, 1] = tau[:, 0] * (a * is2 * np.abs(tt)).sum(1) + S_dhc
    S_g[:, 2:] = tau * a * is2 + np.abs(tt)
    return lp, g, S_lp, S_g


def radon_ref(county, x, y, J, Q, pad=None):
    """``pad[c]``: padding slots of county c in the kernel's rows (their residual -alpha_c enters the sums and is removed)."""
    idx = np.asarray(county, dtype=np.int64)
    x, y, Q = _ld(x), _ld(y), _ld(np.atleast_2d(Q))
    N = len(y)
    pad = np.zeros(J) if pad is None else pad
    padl = _ld(pad)
    mu_a, lsa, mu_b, lsb, le = Q[:, 0], Q[:, 1], Q[:, 2], Q[:, 3], Q[:, 4 + 2 * J]
    a, b = Q[:, 4:4 + J], Q[:, 4 + J:4 + 2 * J]
    sa, sb, eps = np.exp(lsa), np.exp(lsb), np.exp(le)
    ie2 = np.exp(-2 * le)
    al, be = mu_a[:, None] + sa[:, None] * a, mu_b[:, None] + sb[:, None] * b
    A, B = np.abs(mu_a)[:, None] + sa[:, None] * np.abs(a), np.abs(mu_b)[:, None] + sb[:, None] * np.abs(b)
    r = y - (al[:, idx] + be[:, idx] * x)
    m = np.abs(y) + A[:, idx] + B[:, idx] * np.abs(x)
    Z = np.zeros((N, J), dtype=LD)
    Z[np.arange(N), idx] = 1
    Ga, Gb = r @ Z, (r * x) @ Z
    Ma = m @ Z + 2 * padl * A
    Mb = (m * np.abs(x)) @ Z
    M2 = (2 * m * m) @ Z + 2 * padl * A * A
    S2 = (r * r).sum(1)
    hca, dhca, S_hca, S_dhca = _halfcauchy(lsa, sa, 5)
    hcb, dhcb, S_hcb, S_dhcb = _halfcauchy(lsb, sb, 5)
    hce, dhce, S_hce, S_dhce = _halfcauchy(le, eps, 5)
    logS = np.log(LD(10000))
    za, zb = mu_a / 10000, mu_b / 10000
    lp = (-za * za / 2 - HALF_LOG_2PI - logS) + (-zb * zb / 2 - HALF_LOG_2PI - logS) + hca + hcb + hce \
        - (a * a).sum(1) / 2 - J * HALF_LOG_2PI - (b * b).sum(1) / 2 - J * HALF_LOG_2PI - S2 * ie2 / 2 - N * (HALF_LOG_2PI + le)
    g = np.empty(Q.shape, dtype=LD)
    g[:, 0] = ie2 * Ga.sum(1) - mu_a / LD(1e8)
    g[:, 1] = sa * ie2 * (a * Ga).sum(1) + dhca
    g[:, 2] = ie2 * Gb.sum(1) - mu_b / LD(1e8)
    g[:, 3] = sb * ie2 * (b * Gb).sum(1) + dhcb
    g[:, 4:4 + J] = (sa * ie2)[:, None] * Ga - a
    g[:, 4 + J:4 + 2 * J] = (sb * ie2)[:, None] * Gb - b
    g[:, 4 + 2 * J] = dhce + S2 * ie2 - N
    S_lp = za * za / 2 + zb * zb / 2 + 2 * (HALF_LOG_2PI + logS) + S_hca + S_hcb + S_hce + (a * a).sum(1) / 2 \
        + (b * b).sum(1) / 2 + 2 * J * HALF_LOG_2PI + M2.sum(1) * ie2 / 2 + N * (HALF_LOG_2PI + np.abs(le))
    S_g = np.empty(Q.shape, dtype=LD)
    S_g[:, 0] = ie2 * Ma.sum(1) + np.abs(mu_a) / LD(1e8)
    S_g[:, 1] = sa * ie2 * (np.abs(a) * Ma).sum(1) + S_dhca
    S_g[:, 2] = ie2 * Mb.sum(1) + np.abs(mu_b) / LD(1e8)
    S_g[:, 3] = sb * ie2 * (np.abs(b) * Mb).sum(1) + S_dhcb
    S_g[:, 4:4 + J] = (sa * ie2)[:, None] * Ma + np.abs(a)
    S_g[:, 4 + J:4 + 2 * J] = (sb * ie2)[:, None] * Mb + np.abs(b)
    S_g[:, 4 + 2 * J] = S_dhce + M2.sum(1) * ie2 + N
    return lp, g, S_lp, S_g


def _softplus(x):
    return np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x)))


def stochvol_ref(y, Q):
    y, Q = _ld(y), _ld(np.atleast_2d(Q))
    T = len(y)
    mu, z, ls, h = Q[:, :1], Q[:, 1], Q[:, 2], Q[:, 3:]
    ez = np.exp(-np.abs(z))
    s = np.where(z >= 0, 1 / (1 + ez), ez / (1 + ez))
    phi = (2 * s - 1)[:, None]
    dphi_half = ez / ((1 + ez) * (1 + ez))
    sig, is2 = np.exp(ls), np.exp(-2 * ls)
    w = y * y * np.exp(-(mu + h))
    e = h[:, 1:] - phi * h[:, :-1]
    mu0 = mu[:, 0]
    log5, log10 = np.log(LD(5)), np.log(LD(10))
    lp = (-mu0 * mu0 / 50 - HALF_LOG_2PI - log5) + (-2 * _softplus(-z) - z) + (log10 - 10 * sig + ls) \
        + (-h[:, 0] ** 2 / 2 - HALF_LOG_2PI) + (-(e * e).sum(1) * is2 / 2 - (T - 1) * (HALF_LOG_2PI + ls)) \
        + (-w.sum(1) / 2 - T * HALF_LOG_2PI - (T * mu0 + h.sum(1)) / 2)
    g = np.empty(Q.shape, dtype=LD)
    gh = w / 2 - LD(0.5)
    gh[:, 1:] -= e * is2[:, None]
    gh[:, :-1] += phi * is2[:, None] * e
    gh[:, 0] -= h[:, 0]
    g[:, 0] = -mu0 / 25 + w.sum(1) / 2 - LD(T) / 2
    g[:, 1] = (1 - 2 * s) + 2 * dphi_half * is2 * (e * h[:, :-1]).sum(1)
    g[:, 2] = 1 - 10 * sig + (e * e).sum(1) * is2 - (T - 1)
    g[:, 3:] = gh
    W = w * (1 + np.abs(mu) + np.abs(h))
    E = np.abs(h[:, 1:]) + np.abs(h[:, :-1])
    S_h = W / 2 + LD(0.5)
    S_h[:, 1:] += E * is2[:, None]
    S_h[:, :-1] += E * is2[:, None]
    S_h[:, 0] += np.abs(h[:, 0])
    S_g = np.empty(Q.shape, dtype=LD)
    S_g[:, 0] = np.abs(mu0) / 25 + W.sum(1) / 2 + LD(T) / 2
    S_g[:, 1] = np.abs(1 - 2 * s) + 1 + 2 * dphi_half * is2 * (E * np.abs(h[:, :-1])).sum(1)
    S_g[:, 2] = 1 + 10 * sig + 2 * (E * E).sum(1) * is2 + (T - 1)
    S_g[:, 3:] = S_h
    S_lp = mu0 * mu0 / 50 + HALF_LOG_2PI + log5 + 2 * _softplus(-z) + np.abs(z) + log10 + 10 * sig + np.abs(ls) \
        + h[:, 0] ** 2 / 2 + HALF_LOG_2PI + (E * E).sum(1) * is2 + (T - 1) * (HALF_LOG_2PI + np.abs(ls)) + W.sum(1) / 2 \
        + T * HALF_LOG_2PI + (T * np.abs(mu0) + np.abs(h).sum(1)) / 2
    return lp, g, S_lp, S_g


def model_ref(spec, Q):
    """(lp, g, S_lp, S_g, c) of a hand-kind ModelSpec at points Q[C][n]; c the constant of the kernel's bound."""
    d = spec.data
    if spec.name == "eight_schools":
        J = len(d["y"])
        return (*eight_ref(d["y"], d["sigma"], Q), -(-J // 32) + 5 + 20)
    if spec.name == "radon":
        J = spec.meta["n_counties"]
        lay = radon_layout(d["county_idx"], J)
        L = -(-max(lay["rows"]) // 2) + 2 + lay["M"] + -(-lay["E"] // 32)
        return (*radon_ref(d["county_idx"], d["floor"], d["y"], J, Q, lay["pad"]), int(L) + 5 + 20)
    if spec.name == "stochvol":
        return (*stochvol_ref(d["y"], Q), npl_team(spec.n) + 12 + 20)
    raise ValueError(spec.name)


def excess(got, ref, S, c):
    """(err / (c u S), err / (u S)) elementwise; the first <= 1 passes."""
    err = np.abs(_ld(got) - _ld(ref))
    uS = np.maximum(U * _ld(S), np.finfo(np.float64).tiny)
    with np.errstate(invalid="ignore"):
        r = (err / uS).astype(np.float64)
    return r / c, r


# ------------------------------------------------------------------------------------------------------------------------
# model builders: ModelSpec (the hand kind) and the same model as IR
# ------------------------------------------------------------------------------------------------------------------------
def eight_spec(y, sigma):
    from pymc_b200 import models

    J = len(y)
    vars_, n = models._layout([("mu", "mu", 1, None, None), ("tau_log__", "tau", 1, "log", None),
                               ("theta_t", "theta_t", J, None, None)])
    ip = np.zeros(n)
    ip[1] = np.log(5.0)
    return models.ModelSpec(models.KIND_EIGHT_SCHOOLS, n, vars_, data={"y": np.asarray(y, float), "sigma": np.asarray(sigma, float)},
                            meta={"initial_point": ip})


def eight_ir(y, sigma):
    from pymc_b200 import ir

    J = len(y)
    return ir.ModelIR(
        name="eight_schools",
        vars=[ir.Var("mu", "mu", 1), ir.Var("tau_log__", "tau", 1, "log", initial=np.log(5.0)), ir.Var("theta_t", "theta_t", J)],
        priors=[ir.Prior("normal", "mu", (0.0, 5.0)), ir.Prior("halfcauchy", "tau_log__", (5.0,)),
                ir.Prior("normal", "theta_t", (0.0, 1.0))],
        likelihoods=[ir.Likelihood("normal", np.asarray(y, float), [ir.Term([("mu", None)]),
                                                                     ir.Term([("tau_log__", None), ("theta_t", None)])],
                                   sigma=np.asarray(sigma, float))])


def radon_spec(county, x, y, J):
    from pymc_b200 import models

    vars_, n = models._layout([("mu_a", "mu_a", 1, None, None), ("sigma_a_log__", "sigma_a", 1, "log", None),
                               ("mu_b", "mu_b", 1, None, None), ("sigma_b_log__", "sigma_b", 1, "log", None),
                               ("a", "a", J, None, None), ("b", "b", J, None, None), ("eps_log__", "eps", 1, "log", None)])
    ip = np.zeros(n)
    ip[1] = ip[3] = ip[n - 1] = np.log(5.0)
    return models.ModelSpec(models.KIND_RADON, n, vars_,
                            data={"county_idx": np.asarray(county, np.int32), "floor": np.asarray(x, float), "y": np.asarray(y, float)},
                            meta={"n_counties": J, "n_obs": len(y), "initial_point": ip})


def radon_ir(county, x, y, J):
    from pymc_b200 import ir

    l5 = np.log(5.0)
    county = np.asarray(county, np.int32)
    return ir.ModelIR(
        name="radon",
        vars=[ir.Var("mu_a", "mu_a", 1), ir.Var("sigma_a_log__", "sigma_a", 1, "log", initial=l5), ir.Var("mu_b", "mu_b", 1),
              ir.Var("sigma_b_log__", "sigma_b", 1, "log", initial=l5), ir.Var("a", "a", J), ir.Var("b", "b", J),
              ir.Var("eps_log__", "eps", 1, "log", initial=l5)],
        priors=[ir.Prior("normal", "mu_a", (0.0, 1.0e4)), ir.Prior("halfcauchy", "sigma_a_log__", (5.0,)),
                ir.Prior("normal", "mu_b", (0.0, 1.0e4)), ir.Prior("halfcauchy", "sigma_b_log__", (5.0,)),
                ir.Prior("normal", "a", (0.0, 1.0)), ir.Prior("normal", "b", (0.0, 1.0)), ir.Prior("halfcauchy", "eps_log__", (5.0,))],
        likelihoods=[ir.Likelihood("normal", np.asarray(y, float), [
            ir.Term([("mu_a", None)]), ir.Term([("sigma_a_log__", None), ("a", county)]),
            ir.Term([("mu_b", None)], coef=np.asarray(x, float)), ir.Term([("sigma_b_log__", None), ("b", county)], coef=np.asarray(x, float))],
            sigma=ir.Ref("eps_log__"))])


def stochvol_spec(y):
    from pymc_b200 import models

    T = len(y)
    vars_, n = models._layout([("mu", "mu", 1, None, None), ("phi_interval__", "phi", 1, "interval", (-1.0, 1.0)),
                               ("sigma_log__", "sigma", 1, "log", None), ("h", "h", T, None, None)])
    ip = np.zeros(n)
    ip[2] = np.log(0.1)
    return models.ModelSpec(models.KIND_STOCHVOL, n, vars_, data={"y": np.asarray(y, float)}, meta={"T": T, "initial_point": ip})


def stochvol_ir(y):
    from pymc_b200 import ir

    T = len(y)
    return ir.ModelIR(
        name="stochvol",
        vars=[ir.Var("mu", "mu", 1), ir.Var("phi_interval__", "phi", 1, "interval", (-1.0, 1.0)),
              ir.Var("sigma_log__", "sigma", 1, "log", initial=np.log(0.1)), ir.Var("h", "h", T)],
        priors=[ir.Prior("normal", "mu", (0.0, 5.0)), ir.Prior("uniform", "phi_interval__", (-1.0, 1.0)),
                ir.Prior("exponential", "sigma_log__", (10.0,))],
        ar1=[ir.AR1("h", ir.Ref("phi_interval__"), ir.Ref("sigma_log__"), 1.0)],
        likelihoods=[ir.Likelihood("normal_logvar", np.asarray(y, float), [ir.Term([("mu", None)]), ir.Term([("h", None)])])])


# ------------------------------------------------------------------------------------------------------------------------
# data builders and evaluation points
# ------------------------------------------------------------------------------------------------------------------------
def radon_sizes(layout, J, rng):
    """County sizes of a named layout; unless the layout empties it, county J - 1 is the largest."""
    if layout == "skewed":  # geometric sizes with about one county in ten empty
        s = rng.geometric(0.3, J)
        s[rng.random(J) < 0.1] = 0
        s[-1] = s.max() + 3
    elif layout == "empty_ends":  # county 0, county J - 1 and more than 32 others empty: a lane loops over the empties
        s = rng.geometric(0.4, J)
        s[0] = s[-1] = 0
        s[rng.choice(np.arange(1, J - 1), 38, replace=False)] = 0
        s[np.flatnonzero(s)[-1]] += 6
    elif layout == "dominant":  # the real Minnesota data's shape: one county of 116 observations, many of 1-2
        s = np.where(rng.random(J) < 0.5, 1, 2) + (rng.random(J) < 0.2) * rng.integers(1, 15, J)
        s[-1] = 116
    elif layout == "singletons":
        s = np.ones(J, dtype=np.int64)
    elif layout.startswith("mod4_"):
        k = int(layout[-1])
        s = 4 * rng.integers(1 if k == 0 else 0, 5, J) + k
        s[-1] = 4 * 6 + k
    elif layout in ("nonempty32", "nonempty33"):  # exactly one full row, or a second row holding one county
        s = np.zeros(J, dtype=np.int64)
        keep = int(layout[-2:])
        s[np.sort(rng.choice(J - 1, keep - 1, replace=False))] = rng.integers(1, 9, keep - 1)
        s[-1] = 12
    elif layout == "ties":  # long runs of equal sizes: the stable sort decides every lane
        s = rng.choice([3, 3, 5, 5, 7], J)
        s[-1] = 9
    elif layout.startswith("hot"):
        s = _dominant_sizes(_dominant_for_hot(int(layout[-1]), J), J)
    else:
        raise ValueError(layout)
    return np.asarray(s, dtype=np.int64)


def radon_data(sizes, rng, extreme):
    """county, x, y for county sizes; extreme: x ~ U(-30, 30) with |x| = 100 at the last observation of the last non-empty
    county, y = 10^3 + N(0, 3) (residuals cancel at mu_a ~ 10^3); else x ~ U(-1, 1) and y ~ 1.5 + N(0, 0.75)."""
    J = len(sizes)
    county = np.repeat(np.arange(J), sizes)
    rng.shuffle(county)
    last = np.flatnonzero(sizes)[-1]
    at = np.flatnonzero(county == last)[-1]
    county[[at, -1]] = county[[-1, at]]  # one of the last county's observations last in the data
    N = len(county)
    if extreme:
        x = rng.uniform(-30.0, 30.0, N)
        x[-1] = 100.0 * (1 if rng.random() < 0.5 else -1)
        y = 1.0e3 + rng.normal(0.0, 3.0, N)
    else:
        x = rng.uniform(-1.0, 1.0, N)
        y = 1.5 + rng.normal(0.0, 0.3, J)[county] - 0.6 * x + rng.normal(0.0, 0.75, N)
    return county.astype(np.int32), x, y


def radon_points(J, rng, C=6):
    """mu_a ~ 10^3 (the residuals cancel), log-scales in [-8, 8] (point 0 all -8, point 1 all +8), a, b ~ N(0, 1) with
    their largest entries at county J - 1."""
    n = 2 * J + 5
    Q = np.empty((C, n))
    Q[:, 0] = 1.0e3 + rng.normal(0.0, 1.0, C)
    Q[:, 2] = rng.normal(0.0, 1.0, C)
    for k in (1, 3, n - 1):
        Q[:, k] = rng.uniform(-8.0, 8.0, C)
        Q[0, k], Q[1, k] = -8.0, 8.0
    Q[:, 4:4 + 2 * J] = rng.normal(0.0, 1.0, (C, 2 * J))
    Q[:, 3 + J] = 4.0 * np.sign(Q[:, 3 + J] + 0.5)
    Q[:, 3 + 2 * J] = -4.0 * np.sign(Q[:, 3 + 2 * J] + 0.5)
    return Q


def eight_data(J, rng, extreme):
    """extreme: y ~ N(0, 20) with |y| largest at j = J - 1, sigma = 10^U(-2, 3) with 10^-2 and 10^3 both present (the
    smallest at J - 1); else y ~ N(0, 10), sigma ~ U(5, 20)."""
    if not extreme:
        return rng.normal(0.0, 10.0, J), rng.uniform(5.0, 20.0, J)
    y = rng.normal(0.0, 20.0, J)
    y[-1] = 100.0
    sigma = 10.0 ** rng.uniform(-2.0, 3.0, J)
    sigma[0] = 1.0e3
    sigma[-1] = 1.0e-2
    return y, sigma


def eight_points(J, rng, C=6):
    """mu ~ N(0, 5); log tau in [-20, 20] (-20, 20, 0 and three uniform); theta ~ N(0, 1) largest at J - 1."""
    Q = np.empty((C, J + 2))
    Q[:, 0] = rng.normal(0.0, 5.0, C)
    Q[:, 1] = np.concatenate([[-20.0, 20.0, 0.0], rng.uniform(-20.0, 20.0, C - 3)])
    Q[:, 2:] = rng.normal(0.0, 1.0, (C, J))
    Q[:, -1] = 5.0
    return Q


def stochvol_data(T, rng, extreme, seed=4):
    """extreme: |y| = 10^U(-3, 3) with random signs, every seventh y exactly 0, |y| = 10^3 at t = T - 1; else the simulated
    series of models.stochvol with every seventh y exactly 0."""
    if extreme:
        y = 10.0 ** rng.uniform(-3.0, 3.0, T) * np.where(rng.random(T) < 0.5, -1.0, 1.0)
        y[-1] = 1.0e3
    else:
        from pymc_b200 import models

        y = models.stochvol(T, seed).data["y"].copy()
    y[3::7] = 0.0
    return y


ZPHI = (0.0, 10.0, -10.0, 20.0, -20.0, 30.0, -30.0)


def stochvol_points(T, rng):
    """One point per z_phi in {0, +-10, +-20, +-30}; log sigma in [-8, 2] (-8 at the saturated points, whose phi gradient is
    then dominated by its e h / sigma^2 sum); mu + h spanning +-30 with |mu + h| = 30 at t = T - 1."""
    C = len(ZPHI)
    Q = np.empty((C, T + 3))
    Q[:, 0] = rng.uniform(-5.0, 5.0, C)
    Q[:, 1] = ZPHI
    Q[:, 2] = np.where(np.abs(Q[:, 1]) >= 20, -8.0, rng.uniform(-8.0, 2.0, C))
    Q[:, 3:] = rng.uniform(-25.0, 25.0, (C, T))
    Q[:, -1] = np.where(np.arange(C) % 2 == 0, 30.0, -30.0) - Q[:, 0]
    return Q


# ------------------------------------------------------------------------------------------------------------------------
# the cases
# ------------------------------------------------------------------------------------------------------------------------
RADON_J = (1, 13, 14, 29, 30, 61, 62, 93, 94, 125)
RADON_LAYOUTS = [("empty_ends", 94), ("empty_ends", 45), ("dominant", 85), ("singletons", 125), ("mod4_0", 40), ("mod4_1", 40),
                 ("mod4_2", 40), ("mod4_3", 40), ("nonempty32", 45), ("nonempty33", 45), ("ties", 70)]
RADON_CASES = [("skewed", J) for J in RADON_J] + RADON_LAYOUTS + [("hot1", 85), ("hot0", 85)]
EIGHT_J = (1, 30, 31, 33, 62, 63, 126, 127, 190, 191, 254)
STOCHVOL_T = (2, 509, 510, 1021, 1022, 2045, 2046, 3069, 3070, 4093)


def radon_case(layout, J, extreme):
    rng = np.random.default_rng(1000 * J + sum(map(ord, layout)))
    sizes = radon_sizes(layout, J, rng)
    county, x, y = radon_data(sizes, np.random.default_rng(rng.integers(1 << 30) + extreme), extreme)
    return county, x, y


def _kernel_name(spec):
    if spec.name == "stochvol":
        return f"StochVolModel<{npl_team(spec.n)},8>"
    return f"{'EightSchoolsModel' if spec.name == 'eight_schools' else 'RadonModel'}<{npl_warp(spec.n)},1>"


def _record(kernel, case, ratio_uS, extra=None):
    worst = float(np.max(ratio_uS)) if np.all(np.isfinite(ratio_uS)) else float("nan")
    _report(f"models/{kernel}/{case}", dict(max_err_over_uS=worst, **(extra or {})))
    prev = _WORST.get(kernel, 0.0)
    _WORST[kernel] = worst if math.isnan(worst) or worst > prev else prev
    _report("models/worst_err_over_uS", dict(_WORST))


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference against mpmath, the layout replica
# ------------------------------------------------------------------------------------------------------------------------
def _mp_logp(spec, q):
    """The model's log-density from its definition (densities, transforms, Jacobians) at mpmath's working precision."""
    import mpmath as mpm

    mp = mpm.mp
    f = [mpm.mpf(float(v)) if not isinstance(v, mpm.mpf) else v for v in q]
    L2P = mpm.log(2 * mp.pi) / 2

    def normal(x, m, s):
        return -((x - m) / s) ** 2 / 2 - L2P - mpm.log(s)

    def halfcauchy_log(z, beta):  # HalfCauchy(beta) density of x = exp(z) with the Jacobian z
        x = mpm.exp(z)
        return mpm.log(2 / (mp.pi * beta * (1 + (x / beta) ** 2))) + z

    d = spec.data
    if spec.name == "eight_schools":
        y, s = d["y"], d["sigma"]
        mu, lt = f[0], f[1]
        tau = mpm.exp(lt)
        lp = normal(mu, 0, 5) + halfcauchy_log(lt, 5)
        for j in range(len(y)):
            lp += normal(f[2 + j], 0, 1) + normal(mpm.mpf(float(y[j])), mu + tau * f[2 + j], mpm.mpf(float(s[j])))
        return lp
    if spec.name == "radon":
        J = spec.meta["n_counties"]
        sa, sb, eps = mpm.exp(f[1]), mpm.exp(f[3]), mpm.exp(f[4 + 2 * J])
        lp = normal(f[0], 0, 10000) + normal(f[2], 0, 10000)
        lp += halfcauchy_log(f[1], 5) + halfcauchy_log(f[3], 5) + halfcauchy_log(f[4 + 2 * J], 5)
        for c in range(J):
            lp += normal(f[4 + c], 0, 1) + normal(f[4 + J + c], 0, 1)
        for i, c in enumerate(d["county_idx"]):
            m = f[0] + sa * f[4 + c] + (f[2] + sb * f[4 + J + c]) * mpm.mpf(float(d["floor"][i]))
            lp += normal(mpm.mpf(float(d["y"][i])), m, eps)
        return lp
    if spec.name == "stochvol":
        y = d["y"]
        T = len(y)
        mu, z, ls = f[0], f[1], f[2]
        s = 1 / (1 + mpm.exp(-z))
        phi = -1 + 2 * s
        sig = mpm.exp(ls)
        lp = normal(mu, 0, 5)
        lp += -mpm.log(2) + mpm.log(2) + mpm.log(s) + mpm.log(1 - s)  # Uniform(-1, 1) + interval Jacobian log((hi - lo) s (1 - s))
        lp += mpm.log(10) - 10 * sig + ls                             # Exponential(10) + log Jacobian
        h = f[3:]
        lp += normal(h[0], 0, 1)
        for t in range(1, T):
            lp += normal(h[t], phi * h[t - 1], sig)
        for t in range(T):
            lp += normal(mpm.mpf(float(y[t])), 0, mpm.exp((mu + h[t]) / 2))
        return lp
    raise ValueError(spec.name)


def _small_specs():
    """Small cases at the extremes: an empty county and continuous x with y offset 10^3; sigma 10^-2 and 10^3 with log tau
    +-20; an exact zero y, z_phi = +-30, log sigma = -8 and mu + h = +-30."""
    rng = np.random.default_rng(11)
    county = np.array([0, 2, 2, 0, 2], dtype=np.int32)
    x = np.array([-30.0, 12.5, 0.0, 7.25, 100.0])
    y = 1.0e3 + rng.normal(0.0, 3.0, 5)
    rs = radon_spec(county, x, y, 3)
    q_r = np.array([[1.0e3 + 0.3, -8.0, 0.7, 8.0, 0.4, -1.1, 2.0, 0.3, 0.9, -1.5, -8.0],
                    [999.0, 3.0, -0.2, -2.5, -0.6, 0.8, 1.2, -0.4, 0.1, 2.2, 1.5]])
    es = eight_spec(np.array([28.0, -3.0, 100.0]), np.array([1.0e-2, 15.0, 1.0e3]))
    q_e = np.array([[1.0, -20.0, 0.5, -1.0, 5.0], [-2.0, 20.0, -0.3, 1.2, 5.0], [0.5, 0.0, 0.1, 0.2, -0.3]])
    ss = stochvol_spec(np.array([0.0, 1.0e-3, -25.0, 1.0e3]))
    q_s = np.array([[0.5, 30.0, -8.0, -20.0, 11.0, -3.0, 29.5], [-2.0, -30.0, -8.0, 15.0, -14.0, 6.0, -28.0],
                    [1.0, 0.0, 2.0, 0.3, -0.2, 0.1, 0.4], [-1.0, 20.0, -3.0, 2.0, -1.0, 0.5, 3.0]])
    return [(rs, q_r), (es, q_e), (ss, q_s)]


@needs_ld
def test_reference_matches_mpmath_and_central_differences():
    import mpmath as mpm

    for spec, Q in _small_specs():
        lp, g, S_lp, S_g = model_ref(spec, Q)[:4]
        for c in range(Q.shape[0]):
            with mpm.workdps(40):
                want = _mp_logp(spec, Q[c])
                assert abs(mpm.mpf(str(lp[c])) - want) <= mpm.mpf(2) ** -58 * mpm.mpf(str(S_lp[c])), (spec.name, c)
            with mpm.workdps(60):
                h = mpm.mpf(10) ** -18
                base = [mpm.mpf(float(v)) for v in Q[c]]
                for k in range(spec.n):
                    up, dn = list(base), list(base)
                    up[k] += h
                    dn[k] -= h
                    fd = (_mp_logp(spec, up) - _mp_logp(spec, dn)) / (2 * h)
                    assert abs(mpm.mpf(str(g[c, k])) - fd) <= mpm.mpf(2) ** -58 * mpm.mpf(str(S_g[c, k])), (spec.name, c, k)


@needs_ld
def test_reference_sees_the_cancelling_phi_gradient():
    """At z_phi = 30 the phi gradient's factor s (1 - s) written with 1 - s loses about 1e-3 of its value in fp64; the
    reference's e / (1 + e)^2 does not, and the bound c u S cannot absorb the difference."""
    spec, Q = _small_specs()[2]
    lp, g, S_lp, S_g, c = model_ref(spec, Q)
    z = Q[0, 1]
    s = 1.0 / (1.0 + math.exp(-z))
    e = math.exp(-abs(z))
    cancelled, stable = 2.0 * s * (1.0 - s), 2.0 * e / ((1.0 + e) * (1.0 + e))
    assert abs(cancelled / stable - 1) > 1e-4
    rest = float(g[0, 1]) - (1 - 2 * s)
    assert excess([(1 - 2 * s) + rest * cancelled / stable], g[0, 1:2], S_g[0, 1:2], c)[0][0] > 1e3


def test_radon_layout_replica_against_hand_worked_table():
    """Worked by hand from prepare_radon and NutsLaunch (227 KB per CTA, 8 chains, kMaxLevels = 12):
    shared = 512 K + 4 (32 M + round4(M)); hot = the largest level <= 2 with shared + 8 nuts_warp_smem_bytes(NP, hot) fitting."""
    def lay(sizes, J=None):
        J = len(sizes) if J is None else J
        return radon_layout(np.repeat(np.arange(len(sizes)), sizes), J)

    L = lay([3])  # one row of 4, + 4: K = 8; 4096 + 36 * 4
    assert (L["K"], L["M"], L["E"], L["shared"]) == (8, 1, 0, 4240) and list(L["pad"]) == [1]
    assert radon_hot_level(L["shared"], 7) == 2
    L = lay([0, 5, 1, 1, 1, 1] + [0] * 34)  # 35 empty: E = 35; row of 8: K = 12
    assert (L["K"], L["M"], L["E"], L["shared"]) == (12, 1, 35, 6288) and L["pad"][1] == 3 and L["pad"][0] == 0
    L = lay([1] * 33)  # a second row with one lane: M = 2, K = 4 + 4 + 4, seg = (64 + 4) ints
    assert (L["K"], L["M"], L["shared"]) == (12, 2, 6144 + 272)
    # 135 counties, M = 5 rows: 32 nines, 32 nines, 26 nines + 5 sevens + 1 two, 32 twos, 7 twos -> 12 + 12 + 12 + 4 + 4 + 4
    L = lay([7] * 5 + [2] * 40 + [9] * 90)
    assert (L["K"], L["M"], L["rows"]) == (48, 5, [12, 12, 12, 4, 4]) and L["shared"] == 48 * 512 + (160 + 8) * 4
    assert L["pad"][0] == 5 and L["pad"][5] == 10 and L["pad"][6] == 2  # the first two lands in row 2 (stable order)
    # J = 85 (n = 175, NPL 6, NP = 192): per chain 8 / 4 / 2 vectors of 1536 B + 480 B of scalars
    #   dominant 280: K = 280 + 4 + 4 + 4 = 292, shared 149504 + 400 = 149904; hot 2 needs 252048 B, hot 1 202896 B
    #   dominant 370: K = 372 + 8 + 4 = 384, shared 197008; hot 1 needs 250000 B, hot 0 225424 B
    #   dominant 400: K = 412, shared 211344; hot 0 needs 239760 B > 232448 B: refused
    for dom, K, shared, hot in ((280, 292, 149904, 1), (370, 384, 197008, 0), (400, 412, 211344, None)):
        L = lay(list(_dominant_sizes(dom)))
        assert (L["K"], L["shared"]) == (K, shared), dom
        assert radon_hot_level(shared, 175) == hot, dom
    assert nuts_warp_smem_bytes(192, 2, 1) == 12768 and nuts_warp_smem_bytes(256, 1, 8) == 4 * 2048 + 480 + 512 + 3 * 2048
    # the layouts the sampler tests use land on the hot level they are named after
    for hot in (1, 0):
        d = _dominant_for_hot(hot)
        assert radon_hot_level(lay(list(_dominant_sizes(d)))["shared"], 175) == hot
        assert radon_hot_level(lay(list(_dominant_sizes(d - 1)))["shared"], 175) == hot + 1


def test_case_tables_cover_every_instantiation():
    assert {npl_warp(2 * J + 5) for J in RADON_J} == {1, 2, 4, 6, 8}
    assert {npl_warp(J + 2) for J in EIGHT_J} == {1, 2, 4, 6, 8}
    assert {npl_team(T + 3) for T in STOCHVOL_T} == {2, 4, 8, 12, 16}
    for edges, f in ((RADON_J, lambda J: 2 * J + 5), (EIGHT_J, lambda J: J + 2)):
        for a, b in zip(edges, edges[1:]):
            if b == a + 1:
                assert npl_warp(f(a)) != npl_warp(f(b)), (a, b)
    assert npl_warp(2 * 126 + 5) == 0 and npl_warp(255 + 2) == 0 and npl_team(4094 + 3) == 0
    for layout, J in RADON_CASES:
        for extreme in (True, False):
            county, x, y = radon_case(layout, J, extreme)
            lay = radon_layout(county, J)
            assert len(np.unique(county)) == J - lay["E"] and radon_hot_level(lay["shared"], 2 * J + 5) is not None
    lays = {lay_: radon_layout(radon_case(lay_, J, True)[0], J) for lay_, J in RADON_CASES}
    assert lays["empty_ends"]["E"] > 32
    assert lays["nonempty32"]["M"] == 1 and lays["nonempty33"]["M"] == 2
    assert radon_hot_level(lays["hot1"]["shared"], 175) == 1 and radon_hot_level(lays["hot0"]["shared"], 175) == 0


# ------------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------------
def _check_against_ref(spec, ir_model, Q, case):
    """b200_logp_dlogp of the hand kind, batched and point by point, against the reference and the generic IR function."""
    from pymc_b200 import engine

    cm = engine.CompiledModel(spec)
    assert cm.spec.name == spec.name
    lp, g = cm.logp_dlogp(Q)
    for c in range(Q.shape[0]):
        lp1, g1 = cm.logp_dlogp(Q[c])
        assert _bits_equal(lp1, lp[c]) and _bits_equal(g1, g[c]), (case, "batched != single point", c)
    lp_r, g_r, S_lp, S_g, c_hand = model_ref(spec, Q)
    ql, rl = excess(lp, lp_r, S_lp, c_hand)
    qg, rg = excess(g, g_r, S_g, c_hand)
    gen = engine.CompiledModel(ir_model, specialise=False)
    assert gen.spec.name == "ir"
    lp_i, g_i = gen.logp_dlogp(Q)
    N = len(spec.data["y"])
    c_ir = N + spec.n + 20
    qli = np.abs(_ld(lp) - _ld(lp_i)) / np.maximum((c_hand + c_ir) * U * S_lp, np.finfo(float).tiny)
    qgi = np.abs(_ld(g) - _ld(g_i)) / np.maximum((c_hand + c_ir) * U * S_g, np.finfo(float).tiny)
    kernel = _kernel_name(spec)
    _record(kernel, case, np.concatenate([rl, rg.ravel()]),
            dict(c=c_hand, logp_excess=float(np.max(ql)), grad_excess=float(np.max(qg)),
                 worst_grad_entry=int(np.unravel_index(np.argmax(qg), qg.shape)[1]),
                 vs_generic_excess=float(max(np.max(qli), np.max(qgi)))))
    assert np.max(ql) <= 1.0, (case, "logp", float(np.max(ql)))
    assert np.max(qg) <= 1.0, (case, "grad", float(np.max(qg)), np.unravel_index(np.argmax(qg), qg.shape))
    assert np.max(qli) <= 1.0 and np.max(qgi) <= 1.0, (case, "vs generic IR", float(np.max(qli)), float(np.max(qgi)))


def _nuts_against_oracle(spec, eps, case, *, C=2, T=8, seed=3, spread=0.3, max_treedepth=10):
    """Fixed-step NUTS (the SMALL eval) against the oracle sampler: identical tree sizes, positions within 1e-9, and the
    model_logp of every draw bit-equal to b200_logp_dlogp at that draw."""
    from oracle import logp_numpy, nuts_numpy
    from pymc_b200 import engine
    from pymc_b200 import rng as brng

    cm = engine.CompiledModel(spec)
    f = logp_numpy.make_logp(spec)
    n = spec.n
    q0 = spec.initial_point() + np.random.default_rng(seed).uniform(-spread, spread, (C, n))
    step_rngs, pot_rngs, _ = brng.chain_generators(seed, C)
    z = brng.momentum_noise(pot_rngs, T, n)
    res = cm.nuts_run(q0, brng.pack_pcg64(step_rngs), tune=0, draws=T, z=z, mass="diag", adapt_step_size=False,
                      eps0=np.full(C, eps), max_treedepth=max_treedepth, early_max_treedepth=min(8, max_treedepth))
    lp, _ = cm.logp_dlogp(res.draws.reshape(-1, n))
    same_logp = _bits_equal(lp, np.asarray(res.stats["model_logp"]).reshape(-1))
    worst, trees = 0.0, []
    for c in range(C):
        o = nuts_numpy.Oracle(f, nuts_numpy.DiagMass(np.ones(n)), adapt_step_size=False, max_treedepth=max_treedepth,
                               early_max_treedepth=min(8, max_treedepth))
        o.da = nuts_numpy.DualAveraging(eps)
        o.rng, o.tune = step_rngs[c], False
        qs, st = o.run(q0[c], 0, T, z=z[c])
        trees.append((np.asarray(st["tree_size"]).tolist(), np.asarray(res.stats["tree_size"][c]).tolist()))
        worst = max(worst, float(np.max(np.abs(qs - res.draws[c]))) if trees[-1][0] == trees[-1][1] else float("inf"))
    _report(f"models/nuts/{_kernel_name(spec)}/{case}", dict(max_abs_position_diff=worst, model_logp_bit_equal=bool(same_logp),
                                                          tree_sizes=trees[0][1]))
    for c, (want, got) in enumerate(trees):
        assert want == got, (case, c, want, got)
    assert worst <= 1e-9, (case, worst)
    assert same_logp, (case, "model_logp != logp_dlogp")


@needs_ld
@pytest.mark.gpu
@pytest.mark.parametrize("layout,J", RADON_CASES, ids=[f"{lay}-J{J}" for lay, J in RADON_CASES])
def test_radon_against_reference(layout, J):
    county, x, y = radon_case(layout, J, extreme=True)
    Q = radon_points(J, np.random.default_rng(J + 7))
    _check_against_ref(radon_spec(county, x, y, J), radon_ir(county, x, y, J), Q, f"{layout}_J{J}")


@pytest.mark.gpu
@pytest.mark.parametrize("layout,J", RADON_CASES, ids=[f"{lay}-J{J}" for lay, J in RADON_CASES])
def test_radon_nuts_against_oracle(layout, J):
    county, x, y = radon_case(layout, J, extreme=False)
    _nuts_against_oracle(radon_spec(county, x, y, J), 0.02, f"{layout}_J{J}")


@needs_ld
@pytest.mark.gpu
@pytest.mark.parametrize("J", EIGHT_J)
def test_eight_schools_against_reference(J):
    rng = np.random.default_rng(J)
    y, sigma = eight_data(J, rng, extreme=True)
    _check_against_ref(eight_spec(y, sigma), eight_ir(y, sigma), eight_points(J, rng), f"J{J}")


@pytest.mark.gpu
@pytest.mark.parametrize("J", EIGHT_J)
def test_eight_schools_nuts_against_oracle(J):
    y, sigma = eight_data(J, np.random.default_rng(J + 1), extreme=False)
    _nuts_against_oracle(eight_spec(y, sigma), 0.02, f"J{J}")


@needs_ld
@pytest.mark.gpu
@pytest.mark.parametrize("T", STOCHVOL_T)
def test_stochvol_against_reference(T):
    rng = np.random.default_rng(T)
    y = stochvol_data(T, rng, extreme=True)
    _check_against_ref(stochvol_spec(y), stochvol_ir(y), stochvol_points(T, rng), f"T{T}")


@pytest.mark.gpu
@pytest.mark.parametrize("T", STOCHVOL_T)
def test_stochvol_nuts_against_oracle(T):
    y = stochvol_data(T, np.random.default_rng(T + 1), extreme=False)
    _nuts_against_oracle(stochvol_spec(y), 0.01, f"T{T}", T=6, spread=0.1, max_treedepth=6)


# ------------------------------------------------------------------------------------------------------------------------
# GPU: routing of models the hand kernels cannot run
# ------------------------------------------------------------------------------------------------------------------------
def _routing_cases():
    from pymc_b200 import ir as irm

    J = 85
    sizes = _dominant_sizes(400, J)
    county, x, y = radon_data(sizes, np.random.default_rng(5), extreme=False)
    ys, ss = eight_data(300, np.random.default_rng(6), extreme=False)
    big = irm.radon_ir(2000, 200, 1)
    L = big.likelihoods[0]
    return [("radon_n405", big, radon_spec(L.terms[1].factors[1][1], L.terms[2].coef, L.y, 200), "chain-per-warp limit \\(256\\)"),
            ("radon_county400", radon_ir(county, x, y, J), radon_spec(county, x, y, J), "227 KB"),
            ("eight_schools_J300", eight_ir(ys, ss), eight_spec(ys, ss), "chain-per-warp limit \\(256\\)")]


@needs_ld
@pytest.mark.gpu
def test_models_the_hand_kernels_cannot_run_fall_back_to_the_generic_function():
    from pymc_b200 import _lib, engine
    from pymc_b200 import ir as irm

    for case, model, spec, why in _routing_cases():
        assert irm.specialise(model) is not None, case  # the shape is recognised ...
        cm = engine.CompiledModel(model)
        assert cm.spec.name == "ir", case  # ... but the hand kernel refuses it and the generic function runs it
        Q = (radon_points if spec.name == "radon" else eight_points)(spec.meta.get("n_counties", spec.n - 2), np.random.default_rng(2))
        if spec.name == "radon":
            Q[:, 0] = np.random.default_rng(3).normal(0.0, 1.0, len(Q))  # this data sits near 0, not 10^3
        lp, g = cm.logp_dlogp(Q)
        lp_r, g_r, S_lp, S_g = (radon_ref(spec.data["county_idx"], spec.data["floor"], spec.data["y"], spec.meta["n_counties"], Q)
                                if spec.name == "radon" else eight_ref(spec.data["y"], spec.data["sigma"], Q))
        c_ir = len(spec.data["y"]) + spec.n + 20
        ql, rl = excess(lp, lp_r, S_lp, c_ir)
        qg, rg = excess(g, g_r, S_g, c_ir)
        _record("generic IR (fallback)", case, np.concatenate([rl, rg.ravel()]))
        assert np.max(ql) <= 1.0 and np.max(qg) <= 1.0, (case, float(np.max(ql)), float(np.max(qg)))
        # the hand kind named directly is refused when the model is created, with the limit in the message
        with pytest.raises(_lib.B200ShapeError, match=why):
            engine.CompiledModel(spec)
    # the largest models each hand kernel runs are still routed to it
    ys, ss = eight_data(254, np.random.default_rng(1), extreme=False)
    assert engine.CompiledModel(eight_ir(ys, ss)).spec.name == "eight_schools"
    county, x, y = radon_case("hot0", 85, extreme=False)
    assert engine.CompiledModel(radon_ir(county, x, y, 85)).spec.name == "radon"
    assert engine.CompiledModel(irm.radon_ir(600, 125, 1)).spec.name == "radon"
