"""The lock-step contraction kernels against a high-precision reference, at every instantiation, ragged edge and data scale.

Kernels under test (fixed dense mass and the GEMM-shaped models, BASELINE configs #3 and #5):
  * ``gemm_nt_dmma_kernel<WM, NB, 3>`` -- the fp64 DMMA GEMM (``-P q``, ``Sigma g``, ``L^-T z``, ``L z``), all seven
    ``(WM, NB)`` instantiations, chosen per call by ``gemm_nt``'s tile rule (replayed here for the device's SM count);
  * ``half_dot_logp_kernel`` -- the dense Gaussian's logp from ``q . g``;
  * ``logistic_fused_kernel<1|4|16>`` + ``logistic_finish_kernel`` -- the fused fp64 logistic pass (K <= 8, <= 32, <= 128);
  * ``logistic_tc_kernel`` + ``logistic_finish_fm_kernel`` and ``gemm_tc_kernel`` -- the split-fp16 tensor-core mode.

Reference.  Every contraction is redone in ``np.longdouble`` (64-bit significand on x86-64, quad on aarch64) from the model's
data alone (``spec.data`` / ``spec.meta``); sigmoid, softplus and the residual ``y - sigmoid(eta)`` use their stable forms.
Rows of a GEMM are independent, so for large outputs the reference takes a subset of chains that includes the first and the
last chain and both sides of every 16-, 64- and 128-chain tile boundary; the full output is then checked against the same
formulas in fp64 NumPy/BLAS with the sum of both bounds.

Bound.  Each output is a sum of terms t_i; S is the sum of the magnitudes it depends on:
  * ``-P q``: S_j = sum_k |P_jk q_k|  (n terms, m = n + 1);
  * dense Gaussian logp = c + q.g / 2: S = |c| + sum_j |q_j| S_j / 2  (m = 2 n + 8: the gradient's error enters the dot product);
  * logistic gradient G_k = sum_i r_i X_ik - beta_k:  S_k = sum_i |X_ik| (|r_i| + A_i / 4 + 1) + |beta_k|, with
    A_i = sum_k |beta_k X_ik| (eta_i carries an error <= K u A_i, and |sigmoid'| <= 1/4) and the 1 for the residual itself:
    r = y - sigmoid(eta) subtracts a number in (0, 1) from a 0/1 label, so its rounding error is absolute (~u), not relative
    to |r| -- at eta = 30, y = 1 the residual is 9e-14 and fp64 holds it to 5e-17 only  (m = N + K + 16);
  * logistic logp: S = sum_i (A_i + |eta_i| + softplus(eta_i)) + |beta|^2 / 2 + K log(2 pi) / 2  (m = N + 2 K + 16).
fp64 kernels: |kernel - ref| <= m u S + 4 u |ref|, u = 2^-53: the forward-error bound of any summation order, so it cannot be
flaky.  Tensor-core kernels: |kernel - ref| <= 2^-18 S.  Derivation: an operand v is hi + lo in fp16 after an exact
power-of-two scaling that puts its row (column) maximum in [2^14, 2^15), so |v - hi - lo| <= 2^-22 |v| (plus an absolute
floor 2^-39 max|v| for entries whose lo piece is subnormal); a product is hi*hi + hi*lo + lo*hi, each exact in fp32, and the
missing lo*lo is < 2^-22 |product|: 2^-21 S from the operands.  The fp32 accumulator covers one 64-term k-block (GEMM) or
two 128-row slabs (logistic gradient) and is then drained into compensated fp32 / fp64 sums, so fp32 rounding adds
(64..256) * 2^-24 S in the worst case and about sqrt(256) * 2^-24 S = 2^-20 S as the random walk it is; the logistic pass
also forms eta and r in fp32 with ~2^-22 approximations of exp/log.  2^-18 S leaves a factor 2-4 above the sum of those.
Every case writes its largest err / (u S) to the parity report (test_gpu_fullsize._report) before it asserts, and the
report keeps the largest per kernel.

Masking bugs are made visible: every case plants its entry of largest magnitude at a boundary -- the last row of the last
slab, the last real feature column, the last chain of a tile -- so a dropped, duplicated or garbage-padded boundary element
misses the bound by orders of magnitude.
"""
import math

import numpy as np
import pytest

from b200_helpers import discrete_equal
from test_gpu_fullsize import _report

LD = np.longdouble
U = 2.0**-53
TC_TOL = 2.0**-18
HAVE_LD = np.finfo(np.longdouble).nmant >= 63
needs_ld = pytest.mark.skipif(not HAVE_LD, reason="np.longdouble has fewer than 63 significand bits on this platform")

_WORST = {}  # kernel -> largest err / (u S) over the cases run


# ------------------------------------------------------------------------------------------------------------------------
# reference (longdouble or float64: the same formulas)
# ------------------------------------------------------------------------------------------------------------------------
def _sigmoid(x):
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, 1 / (1 + e), e / (1 + e))


def _softplus(x):
    return np.maximum(x, 0) + np.log1p(np.exp(-np.abs(x)))


def _log2pi(dt):
    return np.log(dt(8) * np.arctan(dt(1)))


def logistic_ref(X, y, B, dt=LD):
    """logp, grad and their magnitude sums S of the logistic GLM (beta ~ Normal(0, 1)^K) for chains B[C][K]."""
    Xl, Bl = np.asarray(X, dtype=dt), np.asarray(B, dtype=dt)
    yl = np.asarray(y, dtype=dt)
    K = Xl.shape[1]
    eta = Bl @ Xl.T                                              # [C][N]
    r = np.where(yl == 1, _sigmoid(-eta), -_sigmoid(eta))        # y - sigmoid(eta), no cancellation
    sp = _softplus(eta)
    half_k_log2pi = dt(K) / 2 * _log2pi(dt)
    lp = (yl * eta - sp).sum(1) - (Bl * Bl).sum(1) / 2 - half_k_log2pi
    g = r @ Xl - Bl
    aX = np.abs(Xl)
    A = np.abs(Bl) @ aX.T
    S_g = (np.abs(r) + A / 4 + 1) @ aX + np.abs(Bl)
    S_lp = (A + np.abs(eta) + sp).sum(1) + (Bl * Bl).sum(1) / 2 + half_k_log2pi
    N = Xl.shape[0]
    return lp, g, S_lp, S_g, N + 2 * K + 16, N + K + 16


def gauss_ref(P, logdet_L, Q, dt=LD):
    """logp, grad = -P q and their magnitude sums S of x ~ MvNormal(0, P^-1) for chains Q[C][n]."""
    Pl, Ql = np.asarray(P, dtype=dt), np.asarray(Q, dtype=dt)
    n = Pl.shape[0]
    g = -(Ql @ Pl.T)
    S_g = np.abs(Ql) @ np.abs(Pl.T)
    c = -dt(n) / 2 * _log2pi(dt) - dt(logdet_L)
    lp = c + (Ql * g).sum(1) / 2
    S_lp = abs(c) + (np.abs(Ql) * S_g).sum(1) / 2
    return lp, g, S_lp, S_g, 2 * n + 8, n + 1


def excess(got, ref, S, m, tc=False):
    """(err / bound, err / (u S)) elementwise; err / bound <= 1 passes.  fp64: m u S + 4 u |ref|; tensor cores: 2^-18 S."""
    ref = np.asarray(ref, dtype=LD)
    S = np.asarray(S, dtype=LD)
    err = np.abs(np.asarray(got, dtype=LD) - ref)
    bound = TC_TOL * S if tc else m * U * S + 4 * U * np.abs(ref)
    tiny = np.finfo(np.float64).tiny
    with np.errstate(invalid="ignore", divide="ignore"):
        return (err / np.maximum(bound, tiny)).astype(np.float64), (err / np.maximum(U * S, tiny)).astype(np.float64)


def chain_subset(C):
    """First and last chain and both sides of every 16-, 64- and 128-chain tile boundary."""
    s = {0, C - 1}
    for t in (16, 64, 128):
        for b in range(t, C, t):
            s.update((b - 1, b))
    return np.array(sorted(s))


def gemm_tile(C, n_out, sms):
    """(WM, NB) of gemm_nt_dmma_kernel that gemm_nt (csrc/b200nuts.cu) launches for C chains, n_out outputs and `sms` SMs."""
    wm = 8 if C > 64 else (4 if C > 32 else 2)
    cb = -(-C // (16 * wm))
    best, best_nb = -1.0, 9
    for nb in ((17, 9, 5) if wm == 8 else (9, 5)):
        tiles = cb * -(-n_out // (8 * nb))
        waves = -(-tiles // sms)
        eff = n_out * cb / (waves * sms * 8 * nb) + 1e-3 * nb
        if eff > best:
            best, best_nb = eff, nb
    return wm, best_nb


GEMM_INSTANTIATIONS = {(2, 5), (2, 9), (4, 5), (4, 9), (8, 5), (8, 9), (8, 17)}


def _record(kernel, case, ratio_uS, extra=None):
    worst = float(np.max(ratio_uS)) if np.all(np.isfinite(ratio_uS)) else float("nan")
    _report(f"contractions/{kernel}/{case}", dict(max_err_over_uS=worst, **(extra or {})))
    prev = _WORST.get(kernel, 0.0)
    _WORST[kernel] = worst if math.isnan(worst) or worst > prev else prev  # a NaN, once seen, stays
    _report("contractions/worst_err_over_uS", dict(_WORST))


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the reference, the tile-rule replica and the bound helper
# ------------------------------------------------------------------------------------------------------------------------
@needs_ld
def test_longdouble_reference_matches_mpmath():
    mpmath = pytest.importorskip("mpmath")
    mp = mpmath.mp
    mp.dps = 40
    rng = np.random.default_rng(0)
    X = rng.normal(0, 1, (5, 3))
    X[4] = [30.0, -2.0, 0.5]             # eta ~ 30: the residual of y = 1 is 1e-13
    y = np.array([1, 0, 1, 0, 1], dtype=np.uint8)
    B = rng.normal(0, 1, (2, 3))
    B[1] = [1.0, 0.0, 0.0]
    lp, g, *_ = logistic_ref(X, y, B)
    for c in range(2):
        beta = [mp.mpf(float(v)) for v in B[c]]
        lp_m, g_m = -mp.mpf(3) / 2 * mp.log(2 * mp.pi) - sum(b * b for b in beta) / 2, [-b for b in beta]
        for i in range(5):
            eta = sum(mp.mpf(float(X[i, k])) * beta[k] for k in range(3))
            lp_m += int(y[i]) * eta - mp.log1p(mp.exp(eta))
            r = int(y[i]) - 1 / (1 + mp.exp(-eta))
            for k in range(3):
                g_m[k] += r * mp.mpf(float(X[i, k]))
        assert abs(mp.mpf(str(lp[c])) - lp_m) <= mp.mpf(2) ** -60 * abs(lp_m)
        for k in range(3):
            assert abs(mp.mpf(str(g[c, k])) - g_m[k]) <= mp.mpf(2) ** -60 * (1 + abs(g_m[k]))
    # the residual of the saturated row keeps its relative precision
    r4 = 1 / (1 + mp.exp(sum(mp.mpf(float(X[4, k])) * mp.mpf(float(B[1, k])) for k in range(3))))
    r_ld = _sigmoid(-(np.asarray(X[4], dtype=LD) @ np.asarray(B[1], dtype=LD)))
    assert abs(mp.mpf(str(r_ld)) - r4) <= mp.mpf(2) ** -60 * r4

    P = rng.normal(0, 1, (4, 4))
    Q = rng.normal(0, 1, (3, 4))
    lp, g, *_ = gauss_ref(P, 0.25, Q)
    for c in range(3):
        q = [mp.mpf(float(v)) for v in Q[c]]
        gm = [-sum(mp.mpf(float(P[j, k])) * q[k] for k in range(4)) for j in range(4)]
        lpm = -2 * mp.log(2 * mp.pi) - mp.mpf(0.25) + sum(q[j] * gm[j] for j in range(4)) / 2
        assert abs(mp.mpf(str(lp[c])) - lpm) <= mp.mpf(2) ** -60 * abs(lpm)
        for j in range(4):
            assert abs(mp.mpf(str(g[c, j])) - gm[j]) <= mp.mpf(2) ** -60 * (1 + abs(gm[j]))


def test_gemm_tile_rule_replica():
    """Table worked by hand from gemm_nt's rule: WM from C; among NB in {17, 9, 5} (WM = 8) or {9, 5}, the largest
    useful-work share of whole waves, plus 1e-3 NB."""
    table = {
        (1, 1, 132): (2, 9),        # 1 tile either way: the 1e-3 NB bonus decides
        (15, 31, 132): (2, 9),
        (31, 129, 132): (2, 5),     # 129 / (132 * 40) + 0.005 > 129 / (132 * 72) + 0.009
        (33, 31, 132): (4, 9),
        (40, 300, 132): (4, 5),     # 300 / 5280 + 0.005 = 0.062 > 300 / 9504 + 0.009 = 0.041
        (129, 31, 132): (8, 17),
        (257, 2049, 132): (8, 9),   # 87 tiles of NB = 9 fill one wave: 0.656 > 0.587 (NB = 5, 2 waves) > 0.359
        (256, 10000, 132): (8, 5),  # 500 tiles / 4 waves: 0.947 > 0.702 (NB = 9) > 0.574 (NB = 17)
        (256, 10000, 148): (8, 17), # 148 tiles = one wave of a 148-SM part
    }
    for (C, n, sms), want in table.items():
        assert gemm_tile(C, n, sms) == want, (C, n, sms)


def test_bound_helper_on_hand_sums():
    # 1 + 2^-53 - 1 in fp64 is 0 (round to even); exact value 2^-53; S = 2 + 2^-53, m = 3 terms
    got = (1.0 + 2.0**-53) - 1.0
    q, r = excess(np.array([got]), np.array([LD(2) ** -53]), np.array([LD(2) + LD(2) ** -53]), 3)
    assert got == 0.0 and q[0] <= 1.0 and r[0] == pytest.approx(1.0 / (2 + 2.0**-53), rel=1e-12)
    # a dropped boundary term (here: 3.0 of S = 5) misses the bound by ~1e15
    q, _ = excess(np.array([2.0]), np.array([LD(5)]), np.array([LD(5)]), 4)
    assert q[0] > 1e14
    # the bound is m u S + 4 u |ref|: an error of exactly that passes, twice that fails
    S, ref = LD(10), LD(-3)
    b = 7 * LD(U) * S + 4 * LD(U) * abs(ref)
    assert excess(np.array([ref + b]), np.array([ref]), np.array([S]), 7)[0][0] <= 1.0 + 1e-12
    assert excess(np.array([ref + 2 * b]), np.array([ref]), np.array([S]), 7)[0][0] > 1.9
    # tensor-core bound: 2^-18 S; NaN never passes
    q, _ = excess(np.array([1.0 + 2.0**-19, np.nan]), np.array([LD(1), LD(1)]), np.array([LD(1), LD(1)]), 1, tc=True)
    assert q[0] == pytest.approx(0.5) and not q[1] <= 1.0
    # the chain subset straddles every tile edge
    s = set(chain_subset(300).tolist())
    assert {0, 299, 15, 16, 63, 64, 127, 128, 255, 256} <= s and 17 not in s


# ------------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------------
def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _logistic_model(X, y, tc=False):
    from pymc_b200 import engine, models

    spec = models.ModelSpec(models.KIND_LOGISTIC, X.shape[1], models._layout([("beta", "beta", X.shape[1], None, None)])[0],
                            data={"X": np.ascontiguousarray(X), "y": np.asarray(y, dtype=np.uint8)}, meta={"n_rows": X.shape[0]})
    cm = engine.CompiledModel(spec)
    if tc:
        cm.set_precision("tc_fp16x2")
    return cm


def _gauss_model(P, s=0, tc=False):
    """x ~ MvNormal with precision P; L, Sigma and L^-T are 2^s I, 4^s I and 2^-s I (only P enters logp_dlogp)."""
    from pymc_b200 import engine, models

    n = P.shape[0]
    eye = np.eye(n)
    spec = models.ModelSpec(models.KIND_MVGAUSS, n, models._layout([("x", "x", n, None, None)])[0],
                            data={"L": eye * 2.0**s, "cov": eye * 4.0**s, "prec": np.ascontiguousarray(P), "LinvT": eye * 2.0**-s},
                            meta={"logdet_L": n * s * math.log(2.0)})
    cm = engine.CompiledModel(spec)
    if tc:
        cm.set_precision("tc_fp16x2")
    return cm, spec


def _logistic_data(N, K, C, seed, tile):
    """X ~ N(0, 1) with its largest entry at the last row's last real feature; beta rows ~ N(0, 1/K) so that eta ~ N(0, 1),
    the last chain of every `tile`-chain tile and the last chain three times larger."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, K))
    X[-1, -1] = 16.0 * np.sign(X[-1, -1] or 1.0)
    B = rng.normal(0.0, 1.0 / math.sqrt(K), (C, K))
    B[tile - 1::tile] *= 3.0
    B[-1] *= 3.0
    eta = B[0] @ X.T
    y = (rng.random(N) < 1.0 / (1.0 + np.exp(-eta))).astype(np.uint8)
    return X, y, B


def _check_logistic(cm, X, y, B, kernel, case, tc=False):
    lp, g = cm.logp_dlogp(B)
    C = B.shape[0]
    sub = np.arange(C) if C * X.shape[0] * X.shape[1] <= 4e7 else chain_subset(C)
    lp_r, g_r, S_lp, S_g, m_lp, m_g = logistic_ref(X, y, B[sub])
    qg, rg = excess(g[sub], g_r, S_g, m_g, tc)
    ql, rl = excess(lp[sub], lp_r, S_lp, m_lp, tc)
    full = {}
    if len(sub) < C:  # every chain against the same formulas in fp64 (BLAS), with the sum of both bounds
        lp64, g64, S_lp64, S_g64, *_ = logistic_ref(X, y, B, dt=np.float64)
        full["grad"] = float(np.max(excess(g, g64, S_g64, m_g, tc)[0])) / 2
        full["logp"] = float(np.max(excess(lp, lp64, S_lp64, m_lp, tc)[0])) / 2
    _record(kernel, case, np.concatenate([rg.ravel(), rl]), dict(grad_excess=float(np.max(qg)), logp_excess=float(np.max(ql)),
                                                                chains_vs_longdouble=int(len(sub)), **{f"{k}_excess_all_chains_fp64": v for k, v in full.items()}))
    assert np.max(qg) <= 1.0, (case, "grad", float(np.max(qg)), np.unravel_index(np.argmax(qg), qg.shape))
    assert np.max(ql) <= 1.0, (case, "logp", float(np.max(ql)))
    for k, v in full.items():
        assert v <= 1.0, (case, k, v)


def _check_gauss(cm, spec, Q, kernel, case, tc=False):
    lp, g = cm.logp_dlogp(Q)
    P, logdet = spec.data["prec"], spec.meta["logdet_L"]
    C, n = Q.shape
    sub = np.arange(C) if n < 1000 else chain_subset(C)
    lp_r, g_r, S_lp, S_g, m_lp, m_g = gauss_ref(P, logdet, Q[sub])
    qg, rg = excess(g[sub], g_r, S_g, m_g, tc)
    ql, rl = excess(lp[sub], lp_r, S_lp, m_lp, tc)
    full = {}
    if len(sub) < C:
        lp64, g64, S_lp64, S_g64, *_ = gauss_ref(P, logdet, Q, dt=np.float64)
        full["grad"] = float(np.max(excess(g, g64, S_g64, m_g, tc)[0])) / 2
        full["logp"] = float(np.max(excess(lp, lp64, S_lp64, m_lp, tc)[0])) / 2
    _record(kernel, case, rg.ravel(), dict(grad_excess=float(np.max(qg)), logp_excess=float(np.max(ql)),
                                          chains_vs_longdouble=int(len(sub)), **{f"{k}_excess_all_chains_fp64": v for k, v in full.items()}))
    _record("half_dot_logp_kernel" if not tc else "half_dot_logp_kernel(tc gradient)", case, rl)
    assert np.max(qg) <= 1.0, (case, "grad", float(np.max(qg)), np.unravel_index(np.argmax(qg), qg.shape))
    assert np.max(ql) <= 1.0, (case, "logp", float(np.max(ql)))
    for k, v in full.items():
        assert v <= 1.0, (case, k, v)
    return g


def _gauss_data(n, C, seed, tile=16):
    """Dense P ~ N(0, 1) (symmetrised) with its largest entry at [n-1, n-1] (last output row, last k); q ~ N(0, 1) with
    the last chain of every `tile`-chain tile and the last chain four times larger."""
    rng = np.random.default_rng(seed)
    P = rng.standard_normal((n, n))
    P = 0.5 * (P + P.T)
    P[-1, -1] = 24.0
    Q = rng.standard_normal((C, n))
    Q[tile - 1::tile] *= 4.0
    Q[-1] *= 4.0
    return P, Q


# ------------------------------------------------------------------------------------------------------------------------
# GPU, fp64 path: logistic_fused_kernel<1|4|16>
# ------------------------------------------------------------------------------------------------------------------------
_K_BUCKETS = {1: (1, 5, 8), 4: (9, 17, 31, 32), 16: (33, 64, 65, 127, 128)}
_N_EDGES = (1, 31, 32, 33, 4097)
_C_EDGES = (1, 127, 128, 129, 300)
_LOGI_CASES = [(kb, ks[j % len(ks)], _N_EDGES[j], _C_EDGES[(j + b) % 5])
               for b, (kb, ks) in enumerate(_K_BUCKETS.items()) for j in range(5)]


@needs_ld
@pytest.mark.gpu
@pytest.mark.parametrize("kb,K,N,C", _LOGI_CASES, ids=[f"KB{kb}-K{K}-N{N}-C{C}" for kb, K, N, C in _LOGI_CASES])
def test_logistic_fused_edges(kb, K, N, C):
    X, y, B = _logistic_data(N, K, C, seed=K * 1000 + N + C, tile=128)
    cm = _logistic_model(X, y)
    _check_logistic(cm, X, y, B, f"logistic_fused_kernel<{kb}>", f"K{K}_N{N}_C{C}")


@needs_ld
@pytest.mark.gpu
def test_logistic_fused_more_chain_blocks_than_sms():
    """C = 128 SMs + 1 chains: more chain blocks than SMs, so every chain block gets one row-CTA (gx = 1)."""
    C = 128 * _sms() + 1
    X, y, B = _logistic_data(64, 8, C, seed=7, tile=128)
    _check_logistic(_logistic_model(X, y), X, y, B, "logistic_fused_kernel<1>", f"K8_N64_C{C}_gx1")


@needs_ld
@pytest.mark.gpu
@pytest.mark.parametrize("label", [0, 1])
@pytest.mark.parametrize("K", [8, 20, 100])
def test_logistic_fused_saturated_eta(K, label):
    """Rows scaled so that chain 0 sees eta in {0, +-1e-8, +-30, +-40, +-800}: exp(-|eta|) underflows, the residual of a
    confident row is 1e-13 .. 0, softplus is eta itself; all-0 and all-1 labels."""
    rng = np.random.default_rng(K + label)
    B = rng.normal(0.0, 1.0, (3, K))
    targets = np.array([0.0, 1e-8, -1e-8, 30.0, -30.0, 40.0, -40.0, 800.0, -800.0] * 4)
    X = np.outer(targets, B[0] / (B[0] @ B[0]))
    X[-1, -1] = 2 * np.max(np.abs(X))  # the largest entry at the last row's last feature
    y = np.full(len(targets), label, dtype=np.uint8)
    kb = 1 if K <= 8 else (4 if K <= 32 else 16)
    _check_logistic(_logistic_model(X, y), X, y, B, f"logistic_fused_kernel<{kb}>", f"saturated_K{K}_y{label}")


# ------------------------------------------------------------------------------------------------------------------------
# GPU, fp64 path: gemm_nt_dmma_kernel (all seven instantiations) + half_dot_logp_kernel through the dense Gaussian
# ------------------------------------------------------------------------------------------------------------------------
_GEMM_EDGE_SHAPES = [(1, 1), (31, 15), (33, 17), (31, 33), (33, 47), (1, 65), (31, 129), (129, 31), (65, 63), (301, 129),
                     (33, 257)]
_GEMM_POOL = [(n, C) for n in (1, 31, 33, 129, 301, 1001, 2049, 4095) for C in (1, 15, 17, 31, 33, 47, 63, 65, 129, 257)]


def _gemm_shapes(sms):
    """The edge shapes, plus the first pool shape (odd n, C = 1 or 15 mod 16) that reaches each instantiation they miss."""
    shapes = list(_GEMM_EDGE_SHAPES)
    hit = {gemm_tile(C, n, sms) for n, C in shapes}
    for n, C in sorted(_GEMM_POOL, key=lambda s: s[0] * s[0] + s[0] * s[1]):
        t = gemm_tile(C, n, sms)
        if t not in hit:
            hit.add(t)
            shapes.append((n, C))
    return shapes, hit


@needs_ld
@pytest.mark.gpu
def test_gemm_nt_dmma_every_instantiation():
    shapes, hit = _gemm_shapes(_sms())
    assert hit == GEMM_INSTANTIATIONS, sorted(GEMM_INSTANTIATIONS - hit)
    for n, C in shapes:
        wm, nb = gemm_tile(C, n, _sms())
        P, Q = _gauss_data(n, C, seed=n * 7 + C, tile=16 * wm)
        cm, spec = _gauss_model(P)
        _check_gauss(cm, spec, Q, f"gemm_nt_dmma_kernel<{wm},{nb}>", f"n{n}_C{C}")
    _report("contractions/gemm_nt_dmma_kernel/instantiations_run", sorted(f"<{a},{b}>" for a, b in hit))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [37, 601])
def test_dense_mass_on_persistent_model_matches_reference(n):
    """A fixed dense mass on a persistent-engine model (std_normal): the lock-step path with the model's own logp kernel at
    row stride ld != n (ls_advance_kernel<16> at n > 512) and three GEMMs at new shapes: Sigma g, L^-T z and L z.  Same tree
    statistics as oracle/nuts_numpy.DenseMass and draws within 1e-9."""
    from oracle import logp_numpy, nuts_numpy
    from pymc_b200 import engine, models
    from pymc_b200 import rng as brng

    spec = models.std_normal(n)
    rng = np.random.default_rng(n)
    A = rng.standard_normal((n, n)) * (0.4 / math.sqrt(n))
    cov = np.diag(np.exp(rng.normal(0.0, 0.2, n))) + A @ A.T
    cm = engine.CompiledModel(spec)
    cm.set_dense_mass(cov=cov)
    C, T, eps = 3, 6, 0.35
    q0 = rng.normal(0.0, 1.0, (C, n))
    step_rngs, pot_rngs, _ = brng.chain_generators(n + 3, C)
    z = brng.momentum_noise(pot_rngs, T, n)
    res = cm.nuts_run(q0, brng.pack_pcg64(step_rngs), tune=0, draws=T, z=z, mass="dense", adapt_step_size=False,
                      eps0=np.full(C, eps))
    f = logp_numpy.make_logp(spec)
    for c in range(C):
        o = nuts_numpy.Oracle(f, nuts_numpy.DenseMass(cov), adapt_step_size=False)
        o.da = nuts_numpy.DualAveraging(eps)
        o.rng, o.tune = step_rngs[c], False
        qs, st = o.run(q0[c], 0, T, z=z[c])
        d = {"stat_" + k: np.asarray(v)[None] for k, v in st.items()}
        assert discrete_equal({k: v[c] for k, v in res.stats.items()}, d, 0).all(), (n, c, st["tree_size"], res.stats["tree_size"][c])
        assert np.max(np.abs(qs - res.draws[c])) <= 1e-9, (n, c)


# ------------------------------------------------------------------------------------------------------------------------
# GPU, tensor-core path at data scales 2^s
# ------------------------------------------------------------------------------------------------------------------------
SCALES = (-20, -10, 0, 10, 17)
_TC_LOGI = [(65, 1, 64), (100, 127, 130), (128, 128, 1), (65, 129, 63), (100, 8193, 65), (128, 8193, 130)]
_TC_GEMM = [(1, 1), (63, 127), (64, 128), (65, 129), (129, 1), (300, 129)]


@needs_ld
@pytest.mark.gpu
@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("K,N,C", _TC_LOGI, ids=[f"K{K}-N{N}-C{C}" for K, N, C in _TC_LOGI])
def test_logistic_tc_at_scale(K, N, C, s):
    """X's columns scaled by 2^s and beta by 2^-s: eta, the residuals and the likelihood are unchanged, the gradient's
    data part scales by 2^s."""
    X, y, B = _logistic_data(N, K, C, seed=K + N + C, tile=64)
    X, B = X * 2.0**s, B * 2.0**-s
    _check_logistic(_logistic_model(X, y, tc=True), X, y, B, "logistic_tc_kernel", f"K{K}_N{N}_C{C}_s{s}", tc=True)


@needs_ld
@pytest.mark.gpu
@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("n,C", _TC_GEMM, ids=[f"n{n}-C{C}" for n, C in _TC_GEMM])
def test_gemm_tc_at_scale(n, C, s):
    """L scaled by 2^s, Sigma by 4^s, P by 4^-s and q by 2^s."""
    P, Q = _gauss_data(n, C, seed=n + C, tile=64)
    cm, spec = _gauss_model(P * 4.0**-s, s, tc=True)
    _check_gauss(cm, spec, Q * 2.0**s, "gemm_tc_kernel", f"n{n}_C{C}_s{s}", tc=True)


@pytest.mark.gpu
@pytest.mark.parametrize("n,C", [(65, 129), (300, 129)])
@pytest.mark.parametrize("precision", ["fp64", "tc_fp16x2"])
def test_gauss_gradient_scale_equivariance(n, C, precision):
    """Power-of-two scaling is exact: the gradient at scale s is 2^-s times the gradient at s = 0, bit for bit."""
    P, Q = _gauss_data(n, C, seed=3 * n + C, tile=64)
    g0 = None
    for s in (0,) + tuple(x for x in SCALES if x):
        cm, _ = _gauss_model(P * 4.0**-s, s, tc=precision == "tc_fp16x2")
        g = cm.logp_dlogp(Q * 2.0**s)[1]
        if g0 is None:
            g0 = g
            continue
        bad = np.flatnonzero(g.ravel() != g0.ravel() * 2.0**-s)
        assert bad.size == 0, (precision, s, bad.size, g.ravel()[bad[:3]], (g0.ravel() * 2.0**-s)[bad[:3]])
