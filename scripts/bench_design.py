"""Design-matrix terms against the column form on the generic IR device function.

A GLM whose linear predictor holds X @ beta, written the way ``from_pymc`` lowers ``pm.math.dot(X, beta)`` (one term per
column of X), runs two ways:

    column   ``CompiledModel(ir, specialise=False)``: the IR as written, each column an indexed term
    fused    ``CompiledModel(ir)``: ``ir.fuse_design_columns`` makes the run one team-parallel design term

The two alternate in one process, ``--repeats`` times each, on two workloads: ``logp_dlogp`` at C points and a fixed-step
NUTS run (diagonal unit mass, no tuning).  Times are device times from ``b200_last_kernel_ms``; grad-evals/s is the sum of
tree sizes over the kernel time.  Before timing, both paths are checked to give the same logp and gradient within
1e-13 * sum|loglik_i| and 1e-12 * max(1, |g|_inf).  The card name and power limit are printed from ``nvidia-smi``.

    python scripts/bench_design.py [--repeats 5] [--shapes logistic,negbin,gamma,poisson]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymc_b200 import _lib, engine, ir  # noqa: E402
from pymc_b200 import rng as brng  # noqa: E402
from pymc_b200.ir import Likelihood, ModelIR, Prior, Ref, Term, Var  # noqa: E402

L2_BYTES = 50 * 2**20  # H100 SXM


def column_glm(dist, N, K, seed):
    """b0 + X @ beta with one term per column of X; beta ~ Normal(0, 1); a random alpha for the dispersion families."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, K)) / np.sqrt(K)
    eta = 0.5 + X @ rng.normal(0.0, 1.0, K)
    vars_ = [Var("b0", "b0", 1), Var("beta", "beta", K)]
    priors = [Prior("normal", "b0", (0.0, 2.0)), Prior("normal", "beta", (0.0, 1.0))]
    kw = {}
    if dist == "poisson_log":
        y = rng.poisson(np.exp(eta)).astype(np.float64)
    else:
        vars_.append(Var("alpha_log__", "alpha", 1, "log", initial=np.log(2.0)))
        priors.append(Prior("exponential", "alpha_log__", (0.5,)))
        kw["alpha"] = Ref("alpha_log__")
        mu = np.exp(eta)
        y = rng.negative_binomial(2.0, 2.0 / (mu + 2.0)).astype(np.float64)
    terms = [Term([("b0", None)])] + [Term([("beta", np.full(N, k, dtype=np.int32))], coef=X[:, k].copy()) for k in range(K)]
    return ModelIR(name=f"{dist}-N{N}-K{K}", vars=vars_, priors=priors, likelihoods=[Likelihood(dist, y, terms, **kw)])


# name -> (builder, K, N, logp points, NUTS chains, draws, max tree depth, step size)
SHAPES = {
    "logistic": (lambda: ir.varying_intercept_logistic_ir(n_obs=2000, n_groups=20, n_features=32, seed=3), 32, 2000,
                 1056, 528, 6, 5, 0.1),
    "negbin": (lambda: column_glm("negative_binomial_log", 5000, 96, 5), 96, 5000, 1056, 528, 3, 4, 0.02),
    "gamma": (lambda: ir.gamma_regression_ir(n_obs=1200, n_features=300, seed=7), 300, 1200, 264, 132, 3, 4, 0.02),
    "poisson": (lambda: column_glm("poisson_log", 2000, 1000, 9), 1000, 2000, 264, 132, 2, 3, 0.01),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def check_same(cf, cc, m, Q):
    lf, gf = cf.logp_dlogp(Q)
    lc, gc = cc.logp_dlogp(Q)
    S = np.abs(lc) + 1.0  # a lower bound of sum |pieces|, so the check is at least as strict as the suite's
    lp_err = float(np.max(np.abs(lf - lc) / S))
    g_err = float(np.max(np.max(np.abs(gf - gc), axis=1) / np.maximum(1.0, np.max(np.abs(gc), axis=1))))
    if not (lp_err <= 1e-13 and g_err <= 1e-12):
        raise SystemExit(f"{m.name}: fused and column paths differ: logp {lp_err:.3g}, gradient {g_err:.3g}")
    return lp_err, g_err


def time_logp(cm, Q):
    cm.logp_dlogp(Q)
    ms, _ = _lib.last_kernel_ms()
    return ms


def time_nuts(cm, m, C, draws, depth, eps, seed=1):
    q0 = m.initial_point() + np.random.default_rng(seed).uniform(-0.2, 0.2, (C, m.n))
    step_rngs, _, _ = brng.chain_generators(seed, C)
    res = cm.nuts_run(q0, brng.pack_pcg64(step_rngs), tune=0, draws=draws, mass="diag", adapt_step_size=False,
                      eps0=np.full(C, eps), max_treedepth=depth, early_max_treedepth=depth)
    ms, _ = _lib.last_kernel_ms()
    return ms, int(np.sum(res.stats["tree_size"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for name in args.shapes.split(","):
        build, K, N, P, C, draws, depth, eps = SHAPES[name]
        m = build()
        cf, cc = engine.CompiledModel(m), engine.CompiledModel(m, specialise=False)
        Q = m.initial_point() + np.random.default_rng(2).uniform(-0.3, 0.3, (P, m.n))
        lp_err, g_err = check_same(cf, cc, m, Q)
        team = "cta" if m.n > 256 else "warp"
        t = {"fused": {"logp_ms": [], "nuts_ms": [], "gevals": []}, "column": {"logp_ms": [], "nuts_ms": [], "gevals": []}}
        for _ in range(args.repeats):
            for path, cm in (("column", cc), ("fused", cf)):
                t[path]["logp_ms"].append(time_logp(cm, Q))
                ms, ge = time_nuts(cm, m, C, draws, depth, eps)
                t[path]["nuts_ms"].append(ms)
                t[path]["gevals"].append(ge)
        x_bytes = N * K * 8
        out = {"shape": name, "n": m.n, "N": N, "K": K, "team": team, "check": {"logp_rel": lp_err, "grad_rel": g_err},
               "X_bytes": {"column (coef, index, CSR rowobs and rowptr per column)": N * K * (8 + 4 + 4) + K * (K + 1) * 4,
                           "fused (row-major X + column-major copy)": 2 * x_bytes},
               "fused_X_fits_in_L2": 2 * x_bytes <= L2_BYTES, "logp_points": P, "nuts_chains": C, "draws": draws,
               "max_treedepth": depth, "eps": eps}
        for path in ("column", "fused"):
            lm, nm, ge = (np.array(t[path][k]) for k in ("logp_ms", "nuts_ms", "gevals"))
            out[path] = {"logp_ms": lm.round(3).tolist(), "logp_grad_evals_per_s_median": float(np.median(P / (lm * 1e-3))),
                         "nuts_ms": nm.round(2).tolist(), "nuts_tree_size_sum": ge.tolist(),
                         "nuts_grad_evals_per_s_median": float(np.median(ge / (nm * 1e-3)))}
        out["speedup_logp"] = out["fused"]["logp_grad_evals_per_s_median"] / out["column"]["logp_grad_evals_per_s_median"]
        out["speedup_nuts"] = out["fused"]["nuts_grad_evals_per_s_median"] / out["column"]["nuts_grad_evals_per_s_median"]
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
