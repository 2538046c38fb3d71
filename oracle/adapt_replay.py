"""TEST INFRASTRUCTURE ONLY -- replay of a run's adaptation from the run's own outputs.

Every adaptation rule of the sampler is a deterministic function of quantities a run already returns: dual averaging of
each tuning draw's ``mean_tree_accept``, the diagonal and dense Welford estimators of the accepted positions (the draws,
with ``store_warmup=True``), the exponentially weighted estimators of the draws and their gradients, and the start
energy of each draw, which is 1/2 |z|^2 - logp(previous position) for every mass kind (p . M^-1 p = |z|^2 when
p = L^-T z and v = L L^T p).  Feeding a device run's outputs to the ``nuts_numpy`` classes checks the device's step
sizes, mass matrices and energies at every draw of every chain, for runs of any length, without leaving the chain's own
path (adaptive chains leave any reference path by chaos after a few dozen draws).

These are drivers only: every update rule is the one of ``oracle/nuts_numpy.py``.  The diagonal estimators and dual
averaging are elementwise, so all chains are replayed as one flat vector, which gives the same bits as one chain at a
time; the dense estimator is replayed chain by chain.
"""
from __future__ import annotations

import numpy as np

from .nuts_numpy import DenseAdaptMass, DiagMass, DiagMassExp, DualAveraging


def replay_step_size(accept, tune, eps0, target=0.8, gamma=0.05, k=0.75, t0=10.0, at=()):
    """Dual averaging driven by each draw's ``mean_tree_accept[C, T]``, updated while t < tune (``Oracle.draw``).

    Returns dict(step_size[C, T], step_size_bar[C, T], final_step_size[C], state={i: dict(log_step, log_bar, hbar,
    da_count)} after the first i iterations for every i in ``at``)."""
    accept = np.asarray(accept, dtype=np.float64)
    C, T = accept.shape
    da = DualAveraging(np.array(np.broadcast_to(np.asarray(eps0, dtype=np.float64), (C,))), target, gamma, k, t0)
    step, bar, state = np.empty((C, T)), np.empty((C, T)), {}
    at = set(at)
    for t in range(T):
        if t in at:
            state[t] = _da_state(da, C)
        da.update(accept[:, t], t < tune)
        step[:, t], bar[:, t] = np.exp(da.log_step), np.exp(da.log_bar)
    if T in at:
        state[T] = _da_state(da, C)
    return dict(step_size=step, step_size_bar=bar, final_step_size=np.exp(da.log_bar), state=state)


def _da_state(da, C):
    return dict(log_step=np.array(np.broadcast_to(da.log_step, (C,))), log_bar=np.array(np.broadcast_to(da.log_bar, (C,))),
                hbar=np.array(np.broadcast_to(da.hbar, (C,))), da_count=da.count)


def replay_diag(draws, tune, var0, mean0, weight=10.0, window=101, discard=50, at=()):
    """QuadPotentialDiagAdapt fed the tuning draws ``draws[C, >= tune, n]``; starts at (mean0, var0) with ``weight``.

    Returns dict(final_var[C, n], state={i: the estimator after the first i iterations}) for every i in ``at``; a state
    holds the fields of ``engine.ChainState``: var, fg_n, fg_mean, fg_m2, bg_n, bg_mean, bg_m2, n_samples, window."""
    draws = np.asarray(draws, dtype=np.float64)
    C, _, n = draws.shape
    flat = lambda a: np.array(np.broadcast_to(np.asarray(a, dtype=np.float64), (C, n))).ravel()  # noqa: E731
    m = DiagMass(flat(var0), adapt=True, initial_mean=flat(mean0), initial_weight=weight, adaptation_window=window,
                 discard_window=discard)
    at, state = set(at), {}
    for t in range(tune):
        if t in at:
            state[t] = _diag_state(m, C, n)
        m.update(draws[:, t].ravel(), None, True)
    for i in at:
        if i >= tune:  # nothing adapts after tuning
            state[i] = _diag_state(m, C, n)
    return dict(final_var=m.var.reshape(C, n).copy(), state=state)


def _diag_state(m, C, n):
    return dict(var=m.var.reshape(C, n).copy(), fg_n=m.fg.count, fg_mean=m.fg.mean.reshape(C, n).copy(),
                fg_m2=m.fg.m2.reshape(C, n).copy(), bg_n=m.bg.count, bg_mean=m.bg.mean.reshape(C, n).copy(),
                bg_m2=m.bg.m2.reshape(C, n).copy(), n_samples=m.k, window=m.window)


def replay_dense(draws, tune, var0, mean0, weight=10.0, window=101, multiplier=2.0, update_window=1):
    """QuadPotentialFullAdapt fed the tuning draws of each chain; starts at (mean0, diag(var0)) with ``weight``.

    Returns dict(final_cov[C, n, n], chol_failed_at[C]): the first iteration whose Cholesky factorisation failed, -1 if
    none did."""
    draws = np.asarray(draws, dtype=np.float64)
    C, _, n = draws.shape
    var0 = np.broadcast_to(np.asarray(var0, dtype=np.float64), (C, n))
    mean0 = np.broadcast_to(np.asarray(mean0, dtype=np.float64), (C, n))
    cov, failed = np.empty((C, n, n)), np.full(C, -1)
    for c in range(C):
        m = DenseAdaptMass(n, mean0[c].copy(), np.diag(var0[c]), weight, adaptation_window=window, multiplier=multiplier,
                           update_window=update_window)
        for t in range(tune):
            m.update(draws[c, t], None, True)
            if m.chol_error is not None and failed[c] < 0:
                failed[c] = t
        cov[c] = m.cov
    return dict(final_cov=cov, chol_failed_at=failed)


def replay_diag_grad(draws, grads, tune, alpha=0.02, discard=50, stop=None):
    """QuadPotentialDiagAdaptExp(use_grads=True) fed the tuning draws and their gradients ``grads[C, >= tune, n]``.

    Returns dict(final_var[C, n])."""
    draws, grads = np.asarray(draws, dtype=np.float64), np.asarray(grads, dtype=np.float64)
    C, _, n = draws.shape
    m = DiagMassExp(C * n, alpha=alpha, stop_adaptation=stop, discard_window=discard)
    for t in range(tune):
        m.update(draws[:, t].ravel(), grads[:, t].ravel(), True)
    return dict(final_var=m.var.reshape(C, n).copy())


def start_energy(z, logp_prev):
    """Energy of the start state of each draw: 1/2 |z|^2 - logp(q_{t-1}), for every mass kind."""
    z = np.asarray(z, dtype=np.float64)
    return 0.5 * np.sum(z * z, axis=-1) - np.asarray(logp_prev, dtype=np.float64)
