"""Generates tests/golden/negbin_fixed.npz: the REFERENCE's own NUTS (loaded verbatim by oracle/ref_loader.py) on the NumPy
density of the hierarchical negative-binomial regression with a random dispersion (pymc_b200.ir.negative_binomial_ir,
evaluated by oracle/ir_numpy_families.py).  Fixed step size, unit diagonal mass, 3 chains x 30 draws.

Run where the reference source tree exists (it is not on the GPU machines; tests only read the stored file):

    python -m oracle.make_golden_families

The file has the layout of oracle/make_golden.py's cases, without the momentum noise (regenerated from the chain seeds by
the test loader, as make_golden.shrink() arranges for the large files).
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import ir_numpy_families, ref_loader  # noqa: E402
from oracle.make_golden import OUT, STAT_KEYS  # noqa: E402
from pymc_b200 import ir  # noqa: E402

EPS = 0.04


def run_chain(m, f, q0, seed, draws, eps):
    """One fixed-step chain through the verbatim reference NUTS with QuadPotentialDiag(ones)."""
    n, off = m.n, m.offsets()
    sizes = {v.name: v.size for v in m.vars}
    start = {v.name: q0[off[v.name] : off[v.name] + v.size].copy() for v in m.vars}
    pot = ref_loader.quadpotential().QuadPotentialDiag(np.ones(n))
    step, _ = ref_loader.make_nuts(f, sizes, start, potential=pot, step_rng=0, adapt_step_size=False, step_scale=eps * n**0.25)
    step.setup_chain(np.random.default_rng(seed), 0, draws)
    step.tune = False
    pt, qs, sts, pre_rng, used_eps = start, [], [], [], []
    for _ in range(draws):
        s = step.rng.bit_generator.state["state"]
        pre_rng.append([s["state"] >> 64, s["state"] & (2**64 - 1), s["inc"] >> 64, s["inc"] & (2**64 - 1)])
        pt, st = step.step(pt)
        used_eps.append(float(step.step_size))
        qs.append(np.concatenate([np.ravel(pt[v.name]) for v in m.vars]))
        sts.append(st[0])
    return np.array(qs), sts, np.array(pre_rng, dtype=np.uint64), np.array(used_eps)


def main():
    if not ref_loader.available():
        raise SystemExit("reference not present; golden vectors can only be generated where its source tree exists")
    m = ir.negative_binomial_ir()
    f = ir_numpy_families.make_logp(m)
    rng = np.random.default_rng(81)
    C, draws = 3, 30
    q0s = np.array([m.initial_point() + rng.uniform(-0.3, 0.3, m.n) for _ in range(C)])
    seeds = np.array([1001 + c for c in range(C)])
    Q, ST, PR, UE = [], [], [], []
    for c in range(C):
        q, sts, pre, ue = run_chain(m, f, q0s[c], int(seeds[c]), draws, EPS)
        Q.append(q); ST.append(sts); PR.append(pre); UE.append(ue)
    out = dict(q0=q0s, seeds=seeds, tune=0, draws=draws, adapt=False, dense=False, draws_q=np.array(Q),
               var=np.ones((C, m.n)), eps=np.full(C, EPS), init_var=np.ones((C, m.n)), step_scale=EPS * m.n**0.25,
               final_var=np.ones((C, m.n)), final_step_size=np.full(C, EPS), pre_rng=np.array(PR), used_eps=np.array(UE),
               pre_var=np.ones((C, draws, m.n)))
    for k in STAT_KEYS:
        out["stat_" + k] = np.array([[s[k] for s in sts] for sts in ST])
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "negbin_fixed.npz"), **out)
    ts = out["stat_tree_size"]
    print(f"negbin_fixed: {C} chains x {draws}, grad evals {int(ts.sum())}, mean depth {out['stat_depth'].mean():.2f}, "
          f"mean accept {out['stat_mean_tree_accept'].mean():.3f}, divergences {int(out['stat_diverging'].sum())}")


if __name__ == "__main__":
    main()
