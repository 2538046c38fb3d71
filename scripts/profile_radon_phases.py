"""Where the persistent NUTS kernel spends its cycles on the Radon bench workload, phase by phase.

Builds the engine with ``-DB200_PHASE_CLOCKS`` into a separate library (``B200_OUT``, default
``build/phases/libb200nuts_phases.so``; the in-tree library is not touched), runs the workload ``bench.py`` times
(Radon, 2048 chains x (1000 tune + 1000 draws), adapt_diag, the same starts, streams and momentum seed) and prints, per
phase, the cycles the chains' warps spent in it divided by the number of leapfrogs.  A warp's cycles are its own elapsed
time on the SM (``clock64()`` deltas taken by its first lane), stalls and the time other warps hold the scheduler
included, so the phases add up to the warp's time per leapfrog.  The start-state evaluation of every iteration counts in
``eval``.  The instrumented kernel is slower than the plain one by the clock reads and one fire-and-forget atomic per
mark: use the table for where time goes, and ``bench.py`` for how long it takes.

    python scripts/profile_radon_phases.py [--lib PATH] [--out DIR]

``--lib`` profiles an already built instrumented library instead of building one.  The card name and power limit are
printed with the table, and everything goes to ``DIR/radon_phases.json`` (default: next to the library).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = [
    ("leapfrog", "the two momentum half-steps and the position step of each leapfrog"),
    ("eval", "model evaluation (logp and gradient), start states included"),
    ("energy", "kinetic-energy reduction, energy error, acceptance sums, the leaf as a height-0 subtree"),
    ("merge h=0", "merging two leaves: U-turn dots, multinomial pick"),
    ("merge h>=1", "merging larger subtrees (levels not in shared memory are read from global memory)"),
    ("park", "storing a finished subtree until its sibling is built"),
    ("doubling", "edge loads and stores, top-level pick, full-tree U-turn check"),
    ("iteration", "momentum draw, record of the draw and its stats, step size and mass-matrix adaptation"),
    ("segment", "ticket, waiting for the chain's previous segment, state load and hand-over"),
]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", default=None, help="an instrumented library built with B200_PHASE_CLOCKS=1 ./build.sh")
    ap.add_argument("--out", default=None, help="directory for radon_phases.json (default: the library's)")
    ap.add_argument("--chains", type=int, default=2048)
    ap.add_argument("--tune", type=int, default=1000)
    ap.add_argument("--draws", type=int, default=1000)
    args = ap.parse_args()

    lib_path = args.lib
    if lib_path is None:
        lib_path = os.path.abspath(os.environ.get("B200_OUT", os.path.join(ROOT, "build", "phases", "libb200nuts_phases.so")))
        os.makedirs(os.path.dirname(lib_path), exist_ok=True)
        subprocess.check_call(["bash", os.path.join(ROOT, "build.sh")], cwd=ROOT,
                              env=dict(os.environ, B200_PHASE_CLOCKS="1", B200_OUT=lib_path))
    lib_path = os.path.abspath(lib_path)
    os.environ["B200_LIB"] = lib_path  # read when pymc_b200._lib is imported
    sys.path.insert(0, ROOT)
    import torch

    from pymc_b200 import _lib, engine, models
    from pymc_b200 import rng as brng

    lib = _lib.load()
    if not hasattr(lib, "b200_phase_clocks"):
        raise SystemExit(f"{lib_path} was built without B200_PHASE_CLOCKS")
    lib.b200_phase_clocks.restype = C.c_int
    lib.b200_phase_clocks.argtypes = [C.c_void_p, C.c_int, C.c_int]

    # the bench workload (bench.py: radon), same starts and streams
    spec = models.radon()
    cm = engine.CompiledModel(spec, device=0)
    n, Cn, tune, draws = spec.n, args.chains, args.tune, args.draws
    step_rngs, _, jitter_seeds = brng.chain_generators(20260922, Cn)
    q0 = np.stack([spec.initial_point() + np.random.default_rng(s).uniform(-1, 1, n) for s in jitter_seeds])
    mean0 = np.broadcast_to(q0.mean(axis=0), (Cn, n)).copy()
    q0_d, mean0_d = torch.as_tensor(q0, device="cuda:0"), torch.as_tensor(mean0, device="cuda:0")
    states = brng.pack_pcg64(step_rngs)

    def run(k):
        return cm.nuts_run(q0_d, states.copy(), tune=tune, draws=draws, mean0=mean0_d, store_warmup=False,
                           philox_seed=1000 + k, device_outputs=True, reuse_outputs=True, mass="diag_adapt")

    run(-1)  # module load, buffers
    n_ph = lib.b200_phase_clocks(None, Cn, 1)
    if n_ph != len(PHASES):
        raise SystemExit(f"the library counts {n_ph} phases, this script knows {len(PHASES)}")
    res = run(0)
    torch.cuda.synchronize()
    cyc = np.zeros((Cn, n_ph), dtype=np.uint64)
    if lib.b200_phase_clocks(cyc.ctypes.data, Cn, 0) != n_ph:
        raise SystemExit(_lib.load().b200_last_error().decode())
    grad_evals = int(res.summary["grad_evals"].sum().item())
    leapfrogs = grad_evals - Cn * (tune + draws)
    per = cyc.sum(axis=0).astype(np.float64) / leapfrogs
    name = card()
    print(f"card: {name}")
    print(f"library: {lib_path}")
    print(f"{Cn} chains x ({tune} + {draws}); {leapfrogs} leapfrogs, {grad_evals} grad evals; kernel {res.kernel_ms:.1f} ms")
    print(f"{'phase':<12} {'cycles/leapfrog':>16} {'share':>7}")
    for (ph, _), v in zip(PHASES, per):
        print(f"{ph:<12} {v:16.0f} {100 * v / per.sum():6.1f}%")
    print(f"{'total':<12} {per.sum():16.0f}")
    out_dir = args.out or os.path.dirname(lib_path)
    os.makedirs(out_dir, exist_ok=True)
    rec = {"card": name, "library": lib_path, "chains": Cn, "tune": tune, "draws": draws, "leapfrogs": leapfrogs,
           "grad_evals": grad_evals, "kernel_ms": res.kernel_ms,
           "cycles_per_leapfrog": {ph: float(v) for (ph, _), v in zip(PHASES, per)},
           "phases": {ph: what for ph, what in PHASES}}
    path = os.path.join(out_dir, "radon_phases.json")
    with open(path, "w") as f:
        json.dump(rec, f, indent=1)
    print(f"wrote {path}")


if __name__ == "__main__":
    main()
