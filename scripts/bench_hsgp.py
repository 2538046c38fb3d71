"""What a Gaussian process through spectral (HSGP) terms costs on the generic IR device function.

Three workloads of ``ir.hsgp_regression_ir`` with a Normal likelihood at N = ``--n-obs`` (default 2000):

    expquad_1d   one ExpQuad term, M = 64
    ard_2d       one ExpQuad term over two inputs with one lengthscale each, M = 12 x 12 = 144
    additive     two ExpQuad terms of M = 64 with their own lengthscales and amplitudes

Each is timed against its floor: the same model with the lengthscales and amplitudes fixed to constants, which lowers to a
plain design term X = Phi diag(s) on the code that existed before spectral terms.  The difference is the cost of the
spectral passes (O(M D) per evaluation) against the O(N M) products both share.  Before timing, every path's logp and
gradient must agree with the NumPy oracle (oracle/ir_numpy_hsgp.py) within 1e-12 relative at 16 of the points.  The paths
then alternate ``--repeats`` times over 1024 chains on three measurements: ``logp_dlogp`` at 1024 points, a fixed-step
NUTS run (unit diagonal mass, no tuning) and an adaptive NUTS run (step size and diagonal mass tuned, then kept draws).
Times are device times from ``b200_last_kernel_ms``; grad-evals/s of NUTS is the sum of tree sizes over the kernel time.
The card name and power limit come from ``nvidia-smi``.

    python scripts/bench_hsgp.py [--repeats 3] [--n-obs 2000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import ir_numpy_hsgp  # noqa: E402
from pymc_b200 import _lib, engine, ir  # noqa: E402
from pymc_b200 import rng as brng  # noqa: E402

C = 1024
WORKLOADS = {"expquad_1d": dict(dims=1, m=64), "ard_2d": dict(dims=2, m=12), "additive": dict(dims=1, m=64, additive=True)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def check_oracle(cm, m, Q):
    f = ir_numpy_hsgp.make_logp(m)
    lp, g = cm.logp_dlogp(Q[:16])
    lo, go = np.array([f(q)[0] for q in Q[:16]]), np.array([f(q)[1] for q in Q[:16]])
    lp_err = float(np.max(np.abs(lp - lo) / np.abs(lo)))
    g_err = float(np.max(np.max(np.abs(g - go), axis=1) / np.maximum(1.0, np.max(np.abs(go), axis=1))))
    if not (lp_err <= 1e-12 and g_err <= 1e-12):
        raise SystemExit(f"{m.name}: the device and the oracle differ: logp {lp_err:.3g}, gradient {g_err:.3g}")
    return {"logp_rel": lp_err, "grad_rel": g_err}


def time_logp(cm, Q):
    cm.logp_dlogp(Q)
    ms, _ = _lib.last_kernel_ms()
    return ms


def time_nuts(cm, m, tune, draws, depth, eps, seed=1):
    q0 = m.initial_point() + np.random.default_rng(seed).uniform(-0.2, 0.2, (C, m.n))
    step_rngs, _, _ = brng.chain_generators(seed, C)
    kw = dict(mass="diag", adapt_step_size=False, eps0=np.full(C, eps)) if tune == 0 else dict(store_warmup=True)
    res = cm.nuts_run(q0, brng.pack_pcg64(step_rngs), tune=tune, draws=draws, max_treedepth=depth,
                      early_max_treedepth=depth, **kw)
    ms, _ = _lib.last_kernel_ms()
    return ms, int(np.sum(res.stats["tree_size"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--n-obs", type=int, default=2000)
    ap.add_argument("--draws", type=int, default=20)
    ap.add_argument("--tune", type=int, default=60)
    ap.add_argument("--depth", type=int, default=6)
    ap.add_argument("--eps", type=float, default=0.02)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    models = {}
    for w, kw in WORKLOADS.items():
        models[w] = ir.hsgp_regression_ir("expquad", n_obs=args.n_obs, **kw)
        models[w + "_floor"] = ir.hsgp_regression_ir("expquad", n_obs=args.n_obs, ls="const", amplitude="const", **kw)
    cms, Qs, checks = {}, {}, {}
    for path, m in models.items():
        cms[path] = engine.CompiledModel(m, specialise=False)
        Qs[path] = m.initial_point() + np.random.default_rng(2).uniform(-0.3, 0.3, (C, m.n))
        checks[path] = check_oracle(cms[path], m, Qs[path])
    keys = ("logp_ms", "fixed_ms", "fixed_gevals", "adapt_ms", "adapt_gevals")
    t = {p: {k: [] for k in keys} for p in models}
    for _ in range(args.repeats):
        for path, m in models.items():
            t[path]["logp_ms"].append(time_logp(cms[path], Qs[path]))
            ms, ge = time_nuts(cms[path], m, 0, args.draws, args.depth, args.eps)
            t[path]["fixed_ms"].append(ms)
            t[path]["fixed_gevals"].append(ge)
            ms, ge = time_nuts(cms[path], m, args.tune, args.draws, args.depth, args.eps)
            t[path]["adapt_ms"].append(ms)
            t[path]["adapt_gevals"].append(ge)
    out = {"N": args.n_obs, "chains": C, "draws": args.draws, "tune": args.tune, "max_treedepth": args.depth, "eps": args.eps}
    for path, m in models.items():
        a = {k: np.array(v) for k, v in t[path].items()}
        M = sum(np.shape(tm.coef)[1] for tm in m.likelihoods[0].terms)
        out[path] = {"n": m.n, "M": M, "team": "cta" if m.n > 256 else "warp", "check": checks[path],
                     "logp_ms": a["logp_ms"].round(3).tolist(),
                     "logp_grad_evals_per_s_median": float(np.median(C / (a["logp_ms"] * 1e-3))),
                     "fixed_ms": a["fixed_ms"].round(2).tolist(),
                     "fixed_grad_evals_per_s_median": float(np.median(a["fixed_gevals"] / (a["fixed_ms"] * 1e-3))),
                     "adapt_ms": a["adapt_ms"].round(2).tolist(),
                     "adapt_grad_evals_per_s_median": float(np.median(a["adapt_gevals"] / (a["adapt_ms"] * 1e-3)))}
    for w in WORKLOADS:  # logp_dlogp time of the spectral model over its floor's, same points, same session
        out[w]["logp_time_over_floor_median"] = float(np.median(np.array(t[w]["logp_ms"]) / np.array(t[w + "_floor"]["logp_ms"])))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
