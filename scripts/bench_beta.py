"""What the Beta regression likelihoods cost on the generic IR device function.

    binomial_logit        ``ir.beta_regression_ir("beta_binomial", "const")`` with its likelihood replaced by
                          ``binomial_logit`` on the same (y, trials, predictor): IrModel, no special function
    beta_binomial_logit   the model as built, constant phi: IrExtendedModel, the out-of-line Beta pass with its rising-factorial
                          sums / lgamma and digamma differences per observation
    beta_const, beta_var  ``ir.beta_regression_ir("beta", "const" | "var")``: lgamma and digamma of a and b per observation

The first two share eta and the slot reduction, so their difference is the cost of the BetaBinomial's special functions
per chain and observation.  Before timing, every path's logp and gradient must agree with the NumPy oracle
(oracle/ir_numpy_beta.py) within 1e-12 relative at 16 of the points.  The paths then alternate ``--repeats`` times on two
workloads over 1024 chains: ``logp_dlogp`` at 1024 points and a fixed-step NUTS run (unit diagonal mass, no tuning).
Times are device times from ``b200_last_kernel_ms``; grad-evals/s of NUTS is the sum of tree sizes over the kernel time.
The card name and power limit come from ``nvidia-smi``.

    python scripts/bench_beta.py [--repeats 5] [--n-obs 2000]
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

from oracle import ir_numpy_beta  # noqa: E402
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


def as_binomial(m):
    """The BetaBinomial model as a Binomial one on the same y, trials and predictor."""
    out = copy.deepcopy(m)
    L = out.likelihoods[0]
    L.dist, L.phi = "binomial_logit", None
    out.name = m.name + "-as-binomial"
    return out


def as_columns(m):
    """The model with its design term written one column per term, the form every layer of the oracle evaluates."""
    out = copy.deepcopy(m)
    for L in out.likelihoods:
        terms = []
        for t in L.terms:
            if ir.is_design(t):
                X = np.asarray(t.coef)
                terms += [ir.Term([(t.factors[0][0], np.full(len(L.y), k, dtype=np.int32))], coef=X[:, k].copy())
                          for k in range(X.shape[1])]
            else:
                terms.append(t)
        L.terms = terms
    return out


def check_oracle(cm, m, Q):
    f = ir_numpy_beta.make_logp(as_columns(m))
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
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    bb = ir.beta_regression_ir("beta_binomial", "const", n_obs=args.n_obs, n_groups=20)
    models = {"binomial_logit": as_binomial(bb), "beta_binomial_logit": bb,
              "beta_const": ir.beta_regression_ir("beta", "const", n_obs=args.n_obs, n_groups=20),
              "beta_var": ir.beta_regression_ir("beta", "var", n_obs=args.n_obs, n_groups=20)}
    cms, Qs, checks = {}, {}, {}
    for path, m in models.items():
        cms[path] = engine.CompiledModel(m, specialise=False)
        Qs[path] = m.initial_point() + np.random.default_rng(2).uniform(-0.3, 0.3, (C, m.n))
        checks[path] = check_oracle(cms[path], m, Qs[path])
    t = {p: {"logp_ms": [], "nuts_ms": [], "gevals": []} for p in models}
    for _ in range(args.repeats):
        for path, m in models.items():
            t[path]["logp_ms"].append(time_logp(cms[path], Qs[path]))
            ms, ge = time_nuts(cms[path], m, args.draws, args.depth, args.eps)
            t[path]["nuts_ms"].append(ms)
            t[path]["gevals"].append(ge)
    out = {"N": args.n_obs, "chains": C, "draws": args.draws, "max_treedepth": args.depth, "eps": args.eps}
    for path, m in models.items():
        lm, nm, ge = (np.array(t[path][k]) for k in ("logp_ms", "nuts_ms", "gevals"))
        out[path] = {"n": m.n, "team": "cta" if m.n > 256 else "warp", "check": checks[path],
                     "kernels": "IrModel" if path == "binomial_logit" else "IrExtendedModel", "logp_ms": lm.round(3).tolist(),
                     "logp_grad_evals_per_s_median": float(np.median(C / (lm * 1e-3))), "nuts_ms": nm.round(2).tolist(),
                     "nuts_tree_size_sum": ge.tolist(), "nuts_grad_evals_per_s_median": float(np.median(ge / (nm * 1e-3)))}
    # the special functions' cost per chain, evaluation and observation: the logp_dlogp time difference
    extra = np.median(np.array(t["beta_binomial_logit"]["logp_ms"]) - np.array(t["binomial_logit"]["logp_ms"]))
    out["beta_binomial_extra_ns_per_chain_obs"] = float(extra * 1e6 / (C * args.n_obs))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
