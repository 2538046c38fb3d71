"""Step sizes, mass matrices and per-draw energies of whole runs, replayed from the runs' own outputs (oracle/adapt_replay.py).

Adaptive chains leave the reference path by chaos after a few dozen draws, so comparisons with goldens stop there.  Every
adaptation rule is, however, a deterministic function of what a run returns: dual averaging of each tuning draw's
mean_tree_accept, the Welford estimators of the accepted positions, and the start energy 1/2 |z|^2 - logp(q_{t-1}).
Replaying those through the nuts_numpy classes checks every draw of every chain of a long device run exactly.

CPU: the replay reproduces the reference's goldens bit for bit (step sizes, pre_var at every draw, final_var, final_cov)
and the energy identity holds on them to rounding.  GPU: long runs of every engine and mass kind against the replay of
their own outputs, and the chain state saved at slice boundaries of the persistent kernel against the replay's state.
"""
import numpy as np
import pytest

from b200_helpers import SPEC_OF, relerr
from oracle import adapt_replay
from pymc_b200 import ir, models

GOLDEN_SPEC = dict(SPEC_OF, eight_schools_full_adapt=models.eight_schools, radon_full_adapt=models.radon,
                   eight_schools_hmc_adapt=models.eight_schools, radon_hmc_adapt=models.radon,
                   eight_schools_adapt_grad=models.eight_schools, radon_adapt_grad=models.radon,
                   radon_dense_full_fixed=models.radon, radon_dense_fullinv_fixed=models.radon)


def _golden_logp(name):
    from oracle import logp_numpy

    return logp_numpy.make_logp(GOLDEN_SPEC[name]())


# ------------------------------------------------------------------------------------------------------------------------
# CPU: the replay against the reference's goldens
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["radon_adapt", "eight_schools_adapt", "radon_small_adapt", "radon_full_adapt",
                                  "eight_schools_full_adapt", "eight_schools_hmc_adapt", "radon_hmc_adapt"])
def test_step_size_replay_reproduces_golden(golden, name):
    d = golden(name)
    n = d["q0"].shape[1]
    step_scale = float(d["step_scale"]) if "step_scale" in d else 0.25
    target = 0.65 if "hmc" in name else 0.8
    r = adapt_replay.replay_step_size(d["stat_mean_tree_accept"], int(d["tune"]), step_scale / n**0.25, target)
    assert np.array_equal(r["step_size"], d["stat_step_size"])
    assert np.array_equal(r["step_size_bar"], d["stat_step_size_bar"])
    if "final_step_size" in d:
        assert np.array_equal(r["final_step_size"], d["final_step_size"])


@pytest.mark.parametrize("name", ["radon_adapt", "eight_schools_adapt", "radon_small_adapt", "eight_schools_warm_adapt",
                                  "radon_warm_adapt", "stochvol_small_adapt", "logistic_small_adapt"])
def test_diag_replay_reproduces_golden_pre_var(golden, name):
    d = golden(name)
    tune, T = int(d["tune"]), int(d["tune"]) + int(d["draws"])
    r = adapt_replay.replay_diag(d["draws_q"], tune, d["init_var"], d["q0"], at=range(T))
    pre_var = np.stack([r["state"][t]["var"] for t in range(T)], axis=1)
    assert np.array_equal(pre_var, d["pre_var"])
    assert np.array_equal(r["final_var"], d["final_var"])


@pytest.mark.parametrize("name", ["eight_schools_full_adapt", "radon_full_adapt"])
def test_dense_replay_reproduces_golden_final_cov(golden, name):
    d = golden(name)
    r = adapt_replay.replay_dense(d["draws_q"], int(d["tune"]), 1.0, d["q0"], window=int(d["adaptation_window"]))
    assert np.all(r["chol_failed_at"] == -1)
    assert np.array_equal(r["final_cov"], d["final_cov"])


@pytest.mark.parametrize("name", ["eight_schools_adapt_grad", "radon_adapt_grad"])
def test_diag_grad_replay_reproduces_golden_final_var(golden, name):
    d = golden(name)
    f = _golden_logp(name)
    grads = np.array([[f(q)[1] for q in chain] for chain in d["draws_q"]])
    r = adapt_replay.replay_diag_grad(d["draws_q"], grads, int(d["tune"]), float(d["alpha"]), int(d["discard_window"]),
                                      int(d["stop_adaptation"]))
    assert np.array_equal(r["final_var"], d["final_var"])


def _identity_residual(E, dE, z, logp_prev):
    """|E - dE - E0| / max(|E|, 1/2 |z|^2 + |logp|) over the draws with finite energies (a diverged HMC trajectory's last
    energy may be infinite)."""
    e0 = adapt_replay.start_energy(z, logp_prev)
    scale = np.maximum(np.abs(E), 0.5 * np.sum(z * z, axis=-1) + np.abs(logp_prev))
    ok = np.isfinite(E) & np.isfinite(dE)
    return float(np.max(np.abs(E - dE - e0)[ok] / scale[ok])) if ok.any() else 0.0


@pytest.mark.parametrize("name", ["std_normal_fixed", "eight_schools_fixed", "eight_schools_adapt", "eight_schools_warm_adapt",
                                  "radon_fixed", "radon_small_adapt", "radon_warm_adapt", "std_normal_team_fixed",
                                  "stochvol_small_adapt", "stochvol_small_fixed", "logistic_small_adapt", "logistic_small_fixed",
                                  "mvgauss_dense_fixed", "mvgauss_dense_stepadapt", "eight_schools_full_adapt",
                                  "radon_full_adapt", "eight_schools_hmc_adapt", "radon_hmc_adapt", "eight_schools_adapt_grad",
                                  "radon_adapt_grad", "radon_dense_full_fixed", "radon_dense_fullinv_fixed"])
def test_energy_identity_on_golden(golden, name):
    """energy - energy_error is the start energy 1/2 |z|^2 - logp(q_{t-1}), whatever the mass matrix."""
    d = golden(name)
    f = _golden_logp(name)
    if "hmc" in name:  # HamiltonianMC reports the logp of the proposal, accepted or not: evaluate the previous position
        q_prev = np.concatenate([d["q0"][:, None], d["draws_q"][:, :-1]], axis=1)
        logp_prev = np.array([[f(q)[0] for q in chain] for chain in q_prev])
    else:
        lp0 = np.array([f(q)[0] for q in d["q0"]])
        logp_prev = np.concatenate([lp0[:, None], d["stat_model_logp"][:, :-1]], axis=1)
    assert _identity_residual(d["stat_energy"], d["stat_energy_error"], d["z"], logp_prev) <= 1e-15


# ------------------------------------------------------------------------------------------------------------------------
# GPU: long device runs against the replay of their own outputs
# ------------------------------------------------------------------------------------------------------------------------
def _handoff_radon_chains():
    """A chain count that makes the persistent Radon kernel hand every chain's state from one warp to another every 100
    iterations (ChainCtx in nuts_warp.cuh).  The kernel keeps 8 chain-warps per CTA resident and runs one CTA per SM;
    three times that many chains still cross the handoff if the occupancy ever doubles."""
    import torch

    return 3 * 8 * torch.cuda.get_device_properties(0).multi_processor_count


# key: (model builder, engine, mass, sampler, chains, tune, draws, extra nuts_run keywords)
CONFIGS = {
    # The bench path: device Philox noise and more chains than resident warps.  At three times the resident chains a
    # 1000 + 100 schedule would need several GB of host draws, so it runs 200 + 20: the handoffs at 100 and 200, the
    # discard boundary and the first window swap.  Longer schedules run below on fewer chains.
    "radon_diag_adapt_philox": (models.radon, "persistent", "diag_adapt", "nuts", None, 200, 20,
                                dict(philox_seed=0x5EED, chain_offset=1000)),
    "eight_schools_diag_adapt": (models.eight_schools, "persistent", "diag_adapt", "nuts", 64, 400, 50, {}),
    "eight_schools_hmc": (models.eight_schools, "persistent", "diag_adapt", "hmc", 64, 600, 50, dict(target_accept=0.65)),
    "radon_diag_adapt_grad": (models.radon, "persistent", "diag_adapt_grad", "nuts", 64, 400, 50, {}),
    "stochvol_cta_diag_adapt": (lambda: models.stochvol(T=100), "persistent", "diag_adapt", "nuts", 64, 500, 50, {}),
    "negbin_ir_warp_diag_adapt": (ir.negative_binomial_ir, "persistent", "diag_adapt", "nuts", 64, 300, 50, {}),
    "negbin_ir_cta_diag_adapt": (ir.negative_binomial_ir, "persistent_team", "diag_adapt", "nuts", 64, 300, 50, {}),
    "logistic_lockstep_diag_adapt": (lambda: models.logistic(n_rows=4096, n_features=8), "lockstep", "diag_adapt", "nuts",
                                     160, 300, 50, {}),
    "mvgauss_dense_step_adapt": (lambda: models.mvgauss(n=60), "lockstep", "dense", "nuts", 40, 200, 30, {}),
    # window 101 doubles to 202: switches at 101 and 303, then the window has grown twice
    "eight_schools_dense_adapt": (models.eight_schools, "lockstep", "dense_adapt", "nuts", 160, 310, 20, {}),
    # multiplier 3: switches at 101 and 404 (303 under a multiplier of 2), covariance refreshed every 5th draw
    "eight_schools_dense_adapt_mult3_upd5": (models.eight_schools, "lockstep", "dense_adapt", "nuts", 16, 410, 20,
                                             dict(window_multiplier=3.0, update_window=5)),
    # A window switch hands the foreground to an estimator that holds only the draws of the last window: with fewer draws
    # than dimensions its covariance is singular, the Cholesky factorisation fails and the chain stops with "Bad initial
    # energy", as in the reference; with barely more draws than dimensions it is still too ill-conditioned (measured: Radon
    # chains stop a few draws after a switch at 180).  So the larger models switch only where the window is over twice n
    # (400 at n = 175, 240 at n = 103), and at n = 300 and 1024 the window is longer than tuning.
    "radon_dense_adapt_window400": (models.radon, "lockstep", "dense_adapt", "nuts", 16, 420, 20,
                                    dict(adaptation_window=400, update_window=5)),
    "stochvol_dense_adapt": (lambda: models.stochvol(T=100), "lockstep", "dense_adapt", "nuts", 16, 260, 20,
                             dict(adaptation_window=240)),
    "negbin_ir_dense_adapt": (ir.negative_binomial_ir, "lockstep", "dense_adapt", "nuts", 16, 250, 20, {}),
    "std_normal_300_dense_adapt": (lambda: models.std_normal(300), "lockstep", "dense_adapt", "nuts", 16, 200, 10,
                                   dict(adaptation_window=400, update_window=1)),
    "std_normal_1024_dense_adapt": (lambda: models.std_normal(1024), "lockstep", "dense_adapt", "nuts", 4, 120, 10,
                                    dict(adaptation_window=2000, update_window=10)),
}


def _oracle_logp(model):
    if isinstance(model, ir.ModelIR):
        from oracle import ir_numpy_families

        return ir_numpy_families.make_logp(model)
    from oracle import logp_numpy

    return logp_numpy.make_logp(model)


def _logp_rows(cm, q):
    """cm.logp_dlogp over q[C, T, n], a block of iterations at a time (the gradients are dropped)."""
    C, T, n = q.shape
    out = np.empty((C, T))
    step = max(1, (1 << 22) // max(1, C * n))
    for t in range(0, T, step):
        out[:, t:t + step] = cm.logp_dlogp(q[:, t:t + step].reshape(-1, n))[0].reshape(C, -1)
    return out


def _invariants(res, draws, q0, tune, sampler, Emax=1000.0, max_td=10, early_td=8):
    """{name: holds?} for the invariants of the per-draw statistics."""
    st = res.stats
    C, T = st["depth"].shape
    q_prev = np.concatenate([q0[:, None], draws[:, :-1]], axis=1)
    stayed = np.all(draws == q_prev, axis=-1)
    idx, size, depth = st["index_in_trajectory"], st["tree_size"], st["depth"]
    acc = st["mean_tree_accept"]
    mee, ee, div = st["max_energy_error"], st["energy_error"], st["diverging"].astype(bool)
    ok = {"index_zero_iff_draw_repeated": bool(np.array_equal(idx == 0, stayed)),
          "mean_tree_accept_in_0_1": bool(np.all((acc >= 0) & (acc <= 1)))}
    with np.errstate(invalid="ignore"):
        ok["max_energy_error_over_Emax_is_divergent"] = not bool(np.any((mee >= Emax) & ~div))
        ok["divergent_has_large_energy_error"] = bool(np.all(~div | (np.abs(mee) >= Emax) | ~np.isfinite(mee)))
        if sampler == "nuts":
            ok["index_within_tree_size_within_depth"] = bool(
                np.all((np.abs(idx) <= size) & (size <= 2**depth.astype(np.int64) - 1)))
            ok["energy_error_within_max"] = bool(np.all((np.abs(ee) <= np.abs(mee)) | ~np.isfinite(mee)))
            ok["depth_within_limits"] = bool(np.all(depth[:, :min(tune, 200)] <= early_td) and np.all(depth <= max_td))
            hit = st["reached_max_treedepth"].astype(bool)
            t = np.arange(T)[None, :]
            ok["reached_max_treedepth_only_after_tuning_at_max"] = bool(np.all(~hit | ((t >= tune) & (depth == max_td))))
    return ok


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(CONFIGS))
def test_gpu_run_matches_replay_of_its_own_outputs(key, monkeypatch):
    from pymc_b200 import engine
    from pymc_b200 import rng as brng
    from test_gpu_fullsize import _report

    build, eng, mass, sampler, C, tune, draws, kw = CONFIGS[key]
    model = build()
    if eng == "persistent_team":
        monkeypatch.setenv("B200_FORCE_TEAM", "1")
    cm = engine.CompiledModel(model)
    n, T = cm.n, tune + draws
    C = C or _handoff_radon_chains()
    rs = np.random.default_rng(list(CONFIGS).index(key))
    q0 = cm.spec.initial_point()[None] + rs.uniform(-0.5, 0.5, (C, n))
    step_rngs, pot_rngs, _ = brng.chain_generators(17, C)
    philox = "philox_seed" in kw
    z = None if philox else brng.momentum_noise(pot_rngs, T, n)
    # mass="dense": the Gaussian's handle carries its own covariance as the mass matrix
    mkw = dict(mean0=q0) if mass in ("diag_adapt", "dense_adapt") else {}
    res = cm.nuts_run(q0, brng.pack_pcg64(step_rngs), tune=tune, draws=draws, z=z, mass=mass, sampler=sampler,
                      store_warmup=True, constrain=False, **mkw, **kw)
    draws_q, st = res.draws, res.stats
    # every measurement goes to the report before the first assertion, so a failing configuration leaves its evidence
    report = {"chains": C, "tune": tune, "draws": draws, "engine": eng, "mass": mass, "sampler": sampler}

    # 1. no frozen chain, every draw finite
    bad = res.summary["bad_energy_at"]
    report["frozen_chains"] = int(np.sum(bad != -1))
    report["all_draws_finite"] = bool(np.all(np.isfinite(draws_q)))

    # 2. step sizes: dual averaging of the device's own acceptance statistics
    eps0 = 0.25 / n**0.25
    r = adapt_replay.replay_step_size(st["mean_tree_accept"], tune, eps0, kw.get("target_accept", 0.8))
    e_step = max(relerr(st["step_size"], r["step_size"]), relerr(st["step_size_bar"], r["step_size_bar"]),
                 relerr(res.summary["final_step_size"], r["final_step_size"]))
    report["max_step_size_relerr"] = e_step

    # 3. mass matrix: the estimator arithmetic is NumPy's (unfused products and sums, IEEE division, NumPy's order)
    exact, chol_failed = None, np.full(C, -1)
    if mass == "diag_adapt":
        rv = adapt_replay.replay_diag(draws_q, tune, 1.0, q0, window=kw.get("adaptation_window", 101))
        exact = bool(np.array_equal(res.summary["final_var"], rv["final_var"]))
    elif mass == "dense_adapt":
        rv = adapt_replay.replay_dense(draws_q, tune, 1.0, q0, window=kw.get("adaptation_window", 101),
                                       multiplier=kw.get("window_multiplier", 2.0), update_window=kw.get("update_window", 1))
        chol_failed = rv["chol_failed_at"]
        report["replay_cholesky_failures"] = int(np.sum(chol_failed != -1))
        exact = bool(np.array_equal(res.summary["final_cov"], rv["final_cov"]))
    elif mass == "diag_adapt_grad":
        grads = np.stack([cm.logp_dlogp(draws_q[:, t])[1] for t in range(tune)], axis=1)
        rv = adapt_replay.replay_diag_grad(draws_q, grads, tune, discard=50)
        exact = bool(np.array_equal(res.summary["final_var"], rv["final_var"]))
    report["mass_bit_exact"] = exact

    # 4. model_logp: the logp of the recorded draw (HamiltonianMC records the proposal's, accepted or not)
    lp = _logp_rows(cm, draws_q)
    rec = st["index_in_trajectory"] != 0 if sampler == "hmc" else np.ones_like(lp, dtype=bool)
    e_lp = relerr(st["model_logp"][rec], lp[rec])
    report["max_model_logp_relerr_vs_batched_logp"] = e_lp
    f = _oracle_logp(model)
    pick = rs.choice(C * T, size=min(2000, C * T), replace=False)
    flat = draws_q.reshape(C * T, n)
    lp_or = np.array([f(flat[i])[0] for i in pick])
    # relative to max(|logp|, 1): a log density is a sum of terms of order one or larger, so where it cancels to nearly
    # zero both evaluations keep an absolute error of a few ulps of those terms (measured: stochastic volatility at
    # logp = 0.0029, device 3.8e-15 and NumPy 1.8e-14 from the long-double value), which a bare relative error would blow up
    dev = lp.reshape(-1)[pick]
    e_or = float(np.max(np.abs(dev - lp_or) / np.maximum(np.abs(lp_or), 1.0)))
    report["max_model_logp_error_vs_numpy_oracle"] = e_or
    w = int(np.argmax(np.abs(dev - lp_or)))
    report["worst_oracle_point"] = {"device": float(dev[w]), "numpy": float(lp_or[w]), "draw_index": int(pick[w] % T)}

    # 5. energy identity: E - dE = 1/2 |z|^2 - logp(q_{t-1}), q_{-1} = q0
    lp0 = cm.logp_dlogp(q0)[0]
    logp_prev = np.concatenate([lp0[:, None], lp[:, :-1]], axis=1)
    chk = slice(None)
    if philox:  # regenerate the device's noise for 64 of the chains
        chk = slice(0, 64)
        c, t, i = np.ix_(np.arange(64), np.arange(T), np.arange(n))
        zc = brng.philox_normal(kw["philox_seed"], c + kw["chain_offset"], t, i)
    else:
        zc = z
    e_id = _identity_residual(st["energy"][chk], st["energy_error"][chk], zc, logp_prev[chk])
    report["max_energy_identity_residual"] = e_id

    # 6. invariants of the statistics and the gradient count
    inv = _invariants(res, draws_q, q0, tune, sampler)
    report["invariants"] = inv
    extra = 1 if eng == "lockstep" else T
    grad_ok = bool(np.array_equal(res.summary["grad_evals"], st["tree_size"].astype(np.int64).sum(axis=1) + extra))
    report["grad_evals_match"] = grad_ok
    _report("adaptation_replay/" + key, report)

    assert np.all(bad == -1), bad
    assert report["all_draws_finite"]
    assert e_step <= 1e-12, e_step
    assert np.all(chol_failed == -1), chol_failed
    if exact is not None:
        assert exact, key
    # the persistent engine records the logp of the same device function the batched evaluation runs; the lock-step
    # engine sums the model's terms in the order of its batch-width reduction
    assert e_lp <= (1e-13 if eng == "lockstep" else 0.0), e_lp
    assert e_or <= 1e-12, e_or
    # p0 = L^-T z amplifies rounding by the condition number of L under a dense mass
    assert e_id <= (1e-10 if mass.startswith("dense") else 1e-12), e_id
    assert all(inv.values()), inv
    assert grad_ok


@pytest.mark.gpu
def test_gpu_slice_boundaries_carry_the_replayed_state():
    """A Radon run cut into slices (iter_begin / iter_count, save / resume): every saved ChainState equals the replay's
    state after that many iterations.  The cuts sit after the first draw, at the discard boundary (50), around the first
    variance update and window swaps (101, 202, 303) and the change of tree-depth limit (200)."""
    from pymc_b200 import engine
    from pymc_b200 import rng as brng

    spec = models.radon()
    cm = engine.CompiledModel(spec)
    C, n, tune, draws = 64, spec.n, 320, 10
    T = tune + draws
    cuts = [1, 51, 52, 100, 101, 102, 200, 202, 303]
    q0 = spec.initial_point()[None] + np.random.default_rng(5).uniform(-0.5, 0.5, (C, n))
    step_rngs, pot_rngs, _ = brng.chain_generators(23, C)
    states = brng.pack_pcg64(step_rngs)
    z = brng.momentum_noise(pot_rngs, T, n)
    saved, parts, prev = {}, [], None
    for b0, b1 in zip([0] + cuts, cuts + [T]):
        save = engine.ChainState(C, n)
        res = cm.nuts_run(q0, states, tune=tune, draws=draws, z=z[:, b0:b1], mass="diag_adapt", mean0=q0, iter_begin=b0,
                          iter_count=b1 - b0, resume=prev, save=save)
        parts.append(res)
        saved[b1], prev = save, save
    draws_q = np.concatenate([p.draws for p in parts], axis=1)
    stats = {k: np.concatenate([p.stats[k] for p in parts], axis=1) for k in parts[0].stats}
    rd = adapt_replay.replay_diag(draws_q, tune, 1.0, q0, at=cuts)
    rs = adapt_replay.replay_step_size(stats["mean_tree_accept"], tune, 0.25 / n**0.25, at=cuts)
    for b in cuts:
        s, d, a = saved[b], rd["state"][b], rs["state"][b]
        assert np.array_equal(s.q, draws_q[:, b - 1]), b
        # hbar is sums and products only; log_step and log_bar also go through the device's log and pow, which differ
        # from glibc's by ulps
        assert np.array_equal(s.hbar, a["hbar"]) and np.all(s.da_count == a["da_count"]), b
        assert relerr(s.log_step, a["log_step"]) <= 1e-12 and relerr(s.log_bar, a["log_bar"]) <= 1e-12, b
        assert np.all(s.n_samples == d["n_samples"]) and np.all(s.window == d["window"]), b
        assert np.all(s.fg_n == d["fg_n"]) and np.all(s.bg_n == d["bg_n"]), b
        for name in ("var", "fg_mean", "fg_m2", "bg_mean", "bg_m2"):
            assert np.array_equal(getattr(s, name), d[name]), (b, name)
        assert np.array_equal(s.n_grad, stats["tree_size"][:, :b].astype(np.int64).sum(axis=1) + b), b
