"""What a finite mixture costs on the generic IR device function, per observation and component.

For each K in --ks, ``ir.mixture_ir("normal", K, "dirichlet", n_obs=N)`` runs on IrExtendedModel (the mixture pass:
one online-logsumexp pass over the N x K terms, then K team reductions that recompute them for the component gradients).
Beside it, ``plain`` is the one-component model on the same data: mu ~ Normal(0, 10), sigma ~ HalfNormal(2),
y_i ~ Normal(mu, sigma), on IrModel.  Each alternates ``--repeats`` times on two workloads over 1024 chains:
``logp_dlogp`` at 1024 points and a fixed-step NUTS run (unit diagonal mass, no tuning).  Times are device times from
``b200_last_kernel_ms``; grad-evals/s of NUTS is the sum of tree sizes over the kernel time.  ``ns_per_obs_component`` is
the logp_dlogp time per chain, observation and component, and ``over_plain`` the same time relative to the plain pass's time
per observation.  The card name and power limit come from ``nvidia-smi`` in the same call.

    python scripts/bench_mixture.py [--repeats 3] [--n-obs 2000] [--ks 2,3,5,8]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_survival import C, card, time_logp, time_nuts  # noqa: E402
from pymc_b200 import engine, ir  # noqa: E402


def plain(m):
    """The one-component Normal model of the mixture's data."""
    return ir.ModelIR(name="plain_normal", vars=[ir.Var("mu", "mu", 1), ir.Var("sigma_log__", "sigma", 1, "log")],
                      priors=[ir.Prior("normal", "mu", (0.0, 10.0)), ir.Prior("halfnormal", "sigma_log__", (2.0,))],
                      likelihoods=[ir.Likelihood("normal", m.likelihoods[0].y.copy(), [ir.Term([("mu", None)])],
                                                 sigma=ir.Ref("sigma_log__"))])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--n-obs", type=int, default=2000)
    ap.add_argument("--ks", default="2,3,5,8")
    ap.add_argument("--draws", type=int, default=20)
    ap.add_argument("--depth", type=int, default=6)
    ap.add_argument("--eps", type=float, default=0.01)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for K in (int(k) for k in args.ks.split(",")):
        m = ir.mixture_ir("normal", K, "dirichlet", n_obs=args.n_obs)
        p = plain(m)
        cm, cp = engine.CompiledModel(m, specialise=False), engine.CompiledModel(p, specialise=False)
        Qm = m.initial_point() + np.random.default_rng(2).uniform(-0.3, 0.3, (C, m.n))
        Qp = p.initial_point() + np.random.default_rng(2).uniform(-0.3, 0.3, (C, p.n))
        t = {k: {"logp_ms": [], "nuts_ms": [], "gevals": []} for k in ("plain", "mixture")}
        for _ in range(args.repeats):
            for key, c, mm, Q in (("plain", cp, p, Qp), ("mixture", cm, m, Qm)):
                t[key]["logp_ms"].append(time_logp(c, Q))
                ms, ge = time_nuts(c, mm, args.draws, args.depth, args.eps)
                t[key]["nuts_ms"].append(ms)
                t[key]["gevals"].append(ge)
        out = {"K": K, "N": args.n_obs, "n": m.n, "chains": C, "draws": args.draws, "max_treedepth": args.depth, "eps": args.eps}
        for key in ("plain", "mixture"):
            lm, nm, ge = (np.array(t[key][k]) for k in ("logp_ms", "nuts_ms", "gevals"))
            out[key] = {"logp_ms": lm.round(3).tolist(), "logp_ms_median": float(np.median(lm)), "nuts_ms": nm.round(2).tolist(),
                        "nuts_grad_evals_per_s_median": float(np.median(ge / (nm * 1e-3)))}
        per_obs = out["plain"]["logp_ms_median"] * 1e6 / (C * args.n_obs)
        out["ns_per_obs_component"] = out["mixture"]["logp_ms_median"] * 1e6 / (C * args.n_obs * K)
        out["plain_ns_per_obs"] = per_obs
        out["over_plain"] = out["ns_per_obs_component"] / per_obs
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
