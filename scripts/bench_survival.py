"""What the larger IrExtendedModel kernels cost: the plain LogNormal survival model two ways on the generic IR device
function.

``ir.survival_regression_ir("lognormal", "plain")`` runs as

    lognormal   the IR as built: a ``lognormal`` likelihood, which only IrExtendedModel evaluates (out of line, through
                the censored / truncated pass)
    normal      the same model with y replaced by log y and the likelihood by ``normal``: IrModel, the kernels every
                model without an extended factor runs

The two do the same arithmetic: the LogNormal is the Normal of log y minus log y, a constant.  Before timing, logp must
agree within 1e-13 * S (S = |logp| + sum |log y_i|) after adding -sum log y, and the gradients within 1e-12 * max(1,
|g|_inf).  The paths then alternate ``--repeats`` times on two workloads over 1024 chains: ``logp_dlogp`` at 1024 points
and a fixed-step NUTS run (unit diagonal mass, no tuning).  Times are device times from ``b200_last_kernel_ms``;
grad-evals/s of NUTS is the sum of tree sizes over the kernel time.  The right-censored Weibull example's NUTS grad-evals/s
is printed beside them, at its own step size.  The card name and power limit come from ``nvidia-smi``.

    python scripts/bench_survival.py [--repeats 5] [--n-obs 2000]
"""
from __future__ import annotations

import argparse
import copy
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from pymc_b200 import _lib, engine, ir  # noqa: E402
from pymc_b200 import rng as brng  # noqa: E402

C = 1024


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def as_normal(m):
    """The LogNormal model as a Normal model of log y."""
    out = copy.deepcopy(m)
    L = out.likelihoods[0]
    L.dist, L.y = "normal", np.log(L.y)
    out.name = m.name + "-as-normal"
    return out


def check_same(c_ln, c_n, sum_log_y, Q):
    l1, g1 = c_ln.logp_dlogp(Q)
    l2, g2 = c_n.logp_dlogp(Q)
    S = np.abs(l2) + abs(sum_log_y)
    lp_err = float(np.max(np.abs(l1 - (l2 - sum_log_y)) / S))
    g_err = float(np.max(np.max(np.abs(g1 - g2), axis=1) / np.maximum(1.0, np.max(np.abs(g2), axis=1))))
    if not (lp_err <= 1e-13 and g_err <= 1e-12):
        raise SystemExit(f"lognormal and normal-of-log-y differ: logp {lp_err:.3g}, gradient {g_err:.3g}")
    return lp_err, g_err


def time_logp(cm, Q):
    cm.logp_dlogp(Q)
    ms, _ = _lib.last_kernel_ms()
    return ms


def time_nuts(cm, m, draws, depth, eps, seed=1):
    q0 = m.initial_point() + np.random.default_rng(seed).uniform(-0.2, 0.2, (C, m.n))
    step_rngs, _, _ = brng.chain_generators(seed, C)
    res = cm.nuts_run(q0, brng.pack_pcg64(step_rngs), tune=0, draws=draws, mass="diag", adapt_step_size=False,
                      eps0=np.full(C, eps), max_treedepth=depth, early_max_treedepth=depth)
    ms, _ = _lib.last_kernel_ms()
    return ms, int(np.sum(res.stats["tree_size"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--n-obs", type=int, default=2000)
    ap.add_argument("--draws", type=int, default=20)
    ap.add_argument("--depth", type=int, default=6)
    ap.add_argument("--eps", type=float, default=0.02)
    ap.add_argument("--weibull-eps", type=float, default=0.005)  # 0.02 diverges at the first step from the start point
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    m = ir.survival_regression_ir("lognormal", "plain", n_obs=args.n_obs, n_groups=20)
    mn = as_normal(m)
    c_ln, c_n = engine.CompiledModel(m, specialise=False), engine.CompiledModel(mn, specialise=False)
    Q = m.initial_point() + np.random.default_rng(2).uniform(-0.3, 0.3, (C, m.n))
    lp_err, g_err = check_same(c_ln, c_n, float(np.sum(np.log(m.likelihoods[0].y))), Q)
    t = {p: {"logp_ms": [], "nuts_ms": [], "gevals": []} for p in ("normal", "lognormal")}
    for _ in range(args.repeats):
        for path, cm, mm in (("normal", c_n, mn), ("lognormal", c_ln, m)):
            t[path]["logp_ms"].append(time_logp(cm, Q))
            ms, ge = time_nuts(cm, mm, args.draws, args.depth, args.eps)
            t[path]["nuts_ms"].append(ms)
            t[path]["gevals"].append(ge)
    out = {"model": m.name, "n": m.n, "N": args.n_obs, "team": "cta" if m.n > 256 else "warp", "chains": C,
           "draws": args.draws, "max_treedepth": args.depth, "eps": args.eps, "check": {"logp_rel": lp_err, "grad_rel": g_err}}
    for path in ("normal", "lognormal"):
        lm, nm, ge = (np.array(t[path][k]) for k in ("logp_ms", "nuts_ms", "gevals"))
        out[path] = {"kernels": "IrModel" if path == "normal" else "IrExtendedModel", "logp_ms": lm.round(3).tolist(),
                     "logp_grad_evals_per_s_median": float(np.median(C / (lm * 1e-3))), "nuts_ms": nm.round(2).tolist(),
                     "nuts_tree_size_sum": ge.tolist(), "nuts_grad_evals_per_s_median": float(np.median(ge / (nm * 1e-3)))}
    out["extended_over_base_logp"] = out["lognormal"]["logp_grad_evals_per_s_median"] / out["normal"]["logp_grad_evals_per_s_median"]
    out["extended_over_base_nuts"] = out["lognormal"]["nuts_grad_evals_per_s_median"] / out["normal"]["nuts_grad_evals_per_s_median"]
    print(json.dumps(out), flush=True)
    w = ir.survival_regression_ir("weibull", "right_censored", n_obs=args.n_obs, n_groups=20)
    cw = engine.CompiledModel(w, specialise=False)
    runs = [time_nuts(cw, w, args.draws, args.depth, args.weibull_eps) for _ in range(args.repeats)]
    print(json.dumps({"model": w.name, "n": w.n, "N": args.n_obs, "chains": C, "draws": args.draws,
                      "max_treedepth": args.depth, "eps": args.weibull_eps, "nuts_ms": [round(r[0], 2) for r in runs],
                      "nuts_tree_size_sum": [r[1] for r in runs],
                      "nuts_grad_evals_per_s_median": float(np.median([r[1] / (r[0] * 1e-3) for r in runs]))}), flush=True)


if __name__ == "__main__":
    main()
