"""Generates tests/golden/reference_chains.npz: chains of the verbatim reference sampler (oracle/ref_loader.py) that
tests/test_oracle_vs_reference.py and tests/test_step_seam.py compare the NumPy restatement and the step-method seam with, and
the instance state of the reference QuadPotential objects tests/test_potentials.py maps onto the engine.

    python -m oracle.make_reference_chains      # needs the reference tree (B200_REFERENCE_ROOT)
"""
from __future__ import annotations

import os
import warnings

import numpy as np

from oracle import logp_numpy, ref_loader
from pymc_b200 import models

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_chains.npz")

PORT_CASES = [("eight_schools", False, 0, 25), ("eight_schools", True, 220, 30), ("radon", True, 130, 10), ("std_normal", False, 0, 10)]
PORT_STATS = ("tree_size", "depth", "index_in_trajectory", "energy", "step_size", "step_size_bar", "mean_tree_accept",
              "max_energy_error", "model_logp", "diverging", "energy_error")
DENSE_ADAPT_CASES = [("eight_schools", 130, 10), ("radon", 60, 5)]
DENSE_ADAPT_STATS = ("tree_size", "depth", "index_in_trajectory", "energy", "step_size")
SEAM_STATS = ("depth", "tree_size", "index_in_trajectory", "diverging", "reached_max_treedepth", "divergences", "step_size",
              "step_size_bar", "mean_tree_accept", "energy", "energy_error", "max_energy_error", "model_logp")


def port_key(name, adapt, tune, draws):
    return f"port_{name}_{int(adapt)}_{tune}_{draws}"


def spec_of(name):
    return models.std_normal(40) if name == "std_normal" else models.BUILDERS[name]()


def run_steps(step, start, spec, tune, draws):
    pt, qs, sts = start, [], []
    for i in range(tune + draws):
        if i == tune:
            step.stop_tuning()
        pt, st = step.step(pt)
        qs.append(np.concatenate([np.ravel(pt[v.name]) for v in spec.vars]))
        sts.append(st[0])
    return np.array(qs), sts


def ref_chain(spec, f, q0, seed, tune, draws, adapt):
    qp = ref_loader.quadpotential()
    n = spec.n
    pot = qp.QuadPotentialDiagAdapt(n, q0.copy(), np.ones(n), 10) if adapt else qp.QuadPotentialDiag(np.ones(n))
    start = {v.name: q0[v.offset : v.offset + v.size].copy() for v in spec.vars}
    step, _ = ref_loader.make_nuts(f, spec.var_sizes, start, potential=pot, step_rng=0, adapt_step_size=adapt)
    step.setup_chain(np.random.default_rng(seed), tune, draws)
    if tune == 0:
        step.tune = False
    return run_steps(step, start, spec, tune, draws)


def potential_cases(qp):
    """The reference QuadPotential objects tests/test_potentials.py maps onto the engine: {case: object}."""
    n = 4
    rng = np.random.default_rng(0)
    v, mean = rng.uniform(0.5, 2.0, n), rng.normal(size=n)
    B = rng.normal(size=(n, n))
    cov = B @ B.T + n * np.eye(n)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cases = {
            "diag": qp.QuadPotentialDiag(v),
            "diag_adapt": qp.QuadPotentialDiagAdapt(n, mean, v, 7, adaptation_window=33, discard_window=9),
            "diag_adapt_exp": qp.QuadPotentialDiagAdaptExp(n, mean, alpha=0.03, use_grads=True, stop_adaptation=120),
            "diag_adapt_exp_nostop": qp.QuadPotentialDiagAdaptExp(n, mean, alpha=0.03, use_grads=True),
            "full": qp.QuadPotentialFull(cov),
            "full_inv": qp.QuadPotentialFullInv(cov),
            "full_adapt": qp.QuadPotentialFullAdapt(n, mean, np.diag(v), 10, adaptation_window=40,
                                                    adaptation_window_multiplier=3, update_window=5),
            "full_adapt_nondiag": qp.QuadPotentialFullAdapt(n, mean, cov, 10),
            "diag_adapt_early": qp.QuadPotentialDiagAdapt(n, mean, v, 7, early_update=True),
            "diag_adapt_multiplier": qp.QuadPotentialDiagAdapt(n, mean, v, 7, adaptation_window_multiplier=2),
            "diag_adapt_exp_nograds": qp.QuadPotentialDiagAdaptExp(n, mean, alpha=0.03),
            "diag_n3": qp.QuadPotentialDiag(np.ones(3)),
        }
    # the sampler-level test: Eight Schools (n = 10)
    rng = np.random.default_rng(1)
    mean10, diag10 = rng.normal(size=10), rng.uniform(0.5, 2.0, 10)
    cases["es_diag_adapt"] = qp.QuadPotentialDiagAdapt(10, mean10, diag10, 4, adaptation_window=20, discard_window=5)
    cases["es_diag"] = qp.QuadPotentialDiag(diag10)
    return cases


def potential_state(case, obj):
    """Class name and every numeric / boolean / array attribute of a potential object, as npz entries."""
    out = {f"pot_{case}__class": np.array(type(obj).__name__)}
    for attr, val in vars(obj).items():
        if isinstance(val, (bool, int, float, np.number, np.bool_)) or (isinstance(val, np.ndarray) and val.dtype.kind in "biuf"):
            out[f"pot_{case}__{attr}"] = np.asarray(val)
    return out


def main():
    out = {}
    for case, obj in potential_cases(ref_loader.quadpotential()).items():
        out.update(potential_state(case, obj))
    for name, adapt, tune, draws in PORT_CASES:
        spec = spec_of(name)
        f = logp_numpy.make_logp(spec)
        q0 = spec.initial_point() + np.random.default_rng(1).uniform(-1, 1, spec.n)
        qr, sr = ref_chain(spec, f, q0, 77, tune, draws, adapt)
        key = port_key(name, adapt, tune, draws)
        out[key + "_q"] = qr
        for k in PORT_STATS:
            out[f"{key}_{k}"] = np.array([s[k] for s in sr])

    # QuadPotentialFull, fixed step size
    spec = models.mvgauss(n=15, seed=2)
    f = logp_numpy.make_logp(spec)
    q0 = np.random.default_rng(3).normal(size=15)
    qp = ref_loader.quadpotential()
    start = {"x": q0.copy()}
    step, _ = ref_loader.make_nuts(f, spec.var_sizes, start, potential=qp.QuadPotentialFull(spec.data["cov"]), step_rng=0,
                                   adapt_step_size=False)
    step.setup_chain(np.random.default_rng(5), 0, 12)
    step.tune = False
    out["dense_full_q"] = run_steps(step, start, spec, 0, 12)[0]

    # QuadPotentialFullAdapt
    for name, tune, draws in DENSE_ADAPT_CASES:
        spec = models.BUILDERS[name]()
        n = spec.n
        f = logp_numpy.make_logp(spec)
        q0 = spec.initial_point() + np.random.default_rng(4).uniform(-1, 1, n)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            pot = qp.QuadPotentialFullAdapt(n, q0.copy(), np.eye(n), 10)
        start = {v.name: q0[v.offset : v.offset + v.size].copy() for v in spec.vars}
        step, _ = ref_loader.make_nuts(f, spec.var_sizes, start, potential=pot, step_rng=0, adapt_step_size=True)
        step.setup_chain(np.random.default_rng(91), tune, draws)
        qs, sts = run_steps(step, start, spec, tune, draws)
        key = f"dense_adapt_{name}"
        out[key + "_q"] = qs
        for k in DENSE_ADAPT_STATS:
            out[f"{key}_{k}"] = np.array([s[k] for s in sts])
        out[key + "_cov"] = step.potential._cov
        out[key + "_chol"] = step.potential._chol

    # the step-method protocol (_iter_sample's loop) on the reference NUTS with its default potential
    spec = models.eight_schools()
    f = logp_numpy.make_logp(spec)
    q0 = spec.initial_point() + np.random.default_rng(3).uniform(-1, 1, spec.n)
    start = {v.name: q0[v.offset : v.offset + v.size].copy() for v in spec.vars}
    tune, draws, seed = 60, 25, 20240922
    ref, _ = ref_loader.make_nuts(f, spec.var_sizes, start, step_rng=0)
    ref.setup_chain(np.random.default_rng(seed), tune, draws)
    ref.tune = bool(tune)
    ref.reset_tuning()
    qs, sts = run_steps(ref, dict(start), spec, tune, draws)
    out["seam_q"] = qs
    for k in SEAM_STATS:
        out[f"seam_{k}"] = np.array([s[k] for s in sts])
    state = int(ref.rng.bit_generator.state["state"]["state"])
    out["seam_rng_after"] = np.array([state >> 64, state & (2**64 - 1)], dtype=np.uint64)
    out["seam_stats_keys"] = np.array(sorted(type(ref).stats_dtypes_shapes))
    out["seam_point_keys"] = np.array(sorted(sts[0]))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
