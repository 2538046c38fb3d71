"""Whole-run sampler: the drop-in for PyMC's external-NUTS seam (SURVEY.md 8b, seam B4).

``sample_b200_nuts`` mirrors the signature and return conventions of ``pymc.sampling.jax.sample_jax_nuts``
(pymc/sampling/jax.py:495-517), which is how ``pm.sample(nuts_sampler=...)`` hands a whole run to an
external sampler (``_sample_external_nuts``, pymc/sampling/mcmc.py:372-550).  All chains run in ONE
call on the device; with ``torch.distributed`` initialised the chains are sharded over the ranks
(``pymc_b200.parallel``).  PyMC / PyTensor / ArviZ are not importable in this image, so ``model`` is a
``ModelSpec`` (pymc_b200.models) and the result is a light ``SampleResult`` with the same groups and
names an ``InferenceData`` would carry (posterior, sample_stats, attrs); ``to_arviz()`` converts when
ArviZ is present.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field

import numpy as np

from . import rng as brng
from .engine import CompiledModel
from .ir import ModelIR
from .models import ModelSpec


class SamplingError(RuntimeError):
    """pymc.exceptions.SamplingError: raised for "Bad initial energy" (hmc/base_hmc.py:205-224)."""


# sample_stats names of the external samplers (pymc/sampling/jax.py:267-274, :376-391) from ours
_STAT_RENAME = {
    "diverging": "diverging",
    "energy": "energy",
    "depth": "tree_depth",
    "tree_size": "n_steps",
    "mean_tree_accept": "acceptance_rate",
    "model_logp": "lp",
    "step_size": "step_size",
    "step_size_bar": "step_size_bar",
    "energy_error": "energy_error",
    "max_energy_error": "max_energy_error",
    "index_in_trajectory": "index_in_trajectory",
    "reached_max_treedepth": "reached_max_treedepth",
}


@dataclass
class SampleResult:
    posterior: dict  # rv name -> [chains, draws, ...]
    sample_stats: dict  # stat name -> [chains, draws]
    unconstrained: np.ndarray | None  # [chains, draws, n] (keep_untransformed)
    warmup_posterior: dict | None = None
    warmup_sample_stats: dict | None = None
    attrs: dict = field(default_factory=dict)
    observed_data: dict = field(default_factory=dict)   # groups external samplers are held to (test_mcmc_external.py:78-85)
    constant_data: dict = field(default_factory=dict)
    log_likelihood: dict = field(default_factory=dict)  # observed rv name -> [chains, draws, N] (idata_kwargs["log_likelihood"])

    def groups(self):
        out = ["posterior", "sample_stats"]
        out += [g for g in ("log_likelihood", "observed_data", "constant_data") if getattr(self, g)]
        out += [g for g in ("warmup_posterior", "warmup_sample_stats") if getattr(self, g) is not None]
        return out

    def to_arviz(self):
        import arviz as az  # optional

        return az.from_dict(posterior=self.posterior, sample_stats=self.sample_stats, observed_data=self.observed_data or None,
                            constant_data=self.constant_data or None, log_likelihood=self.log_likelihood or None, attrs=self.attrs)


def _log_likelihood(cm, dq):
    """The `log_likelihood` group (sampling/jax.py:128-144, :660-673; pm.compute_log_likelihood, stats/log_density.py:31-77):
    log p(y_i | draw) for every likelihood factor of the model's IR, evaluated on the device by the generic IR function
    (``b200_pointwise_loglik``).  ``dq``: unconstrained draws [chains, draws, n]."""
    ir = getattr(cm, "ir", None)
    if ir is None or not hasattr(cm, "pointwise_loglik"):
        raise NotImplementedError("idata_kwargs={'log_likelihood': True} needs a model given as pymc_b200.ir.ModelIR (from_pymc)")
    eng = cm
    if getattr(cm.spec, "name", "ir") != "ir":  # the model runs on a hand-specialised kernel: the pointwise pass is the generic one
        eng = cm.__dict__.get("_generic_engine")
        if eng is None:
            eng = cm.__dict__["_generic_engine"] = CompiledModel(ir, device=getattr(cm, "device", None), specialise=False)
    return {L.name: eng.pointwise_loglik(np.asarray(dq), lik=i) for i, L in enumerate(ir.likelihoods)}


def initial_points(spec: ModelSpec, chains: int, jitter_seeds, initvals=None, jitter=True, logp_fn=None,
                   jitter_max_retries=10):
    """Per-chain start = the model's initial point (+ U(-1,1) jitter), re-drawn until logp is finite
    (``_init_jitter``, pymc/sampling/mcmc.py:1695-1756; pymc/initial_point.py:328-340).

    The reference draws the jitter with PyTensor RNG ops reseeded in graph-traversal order, which is
    PyTensor-internal: parity with its jitter is unpinned (SURVEY 8a a17); here each chain's jitter comes
    from ``default_rng(jitter_seed)`` in raveled-vector order.  Pass ``initvals`` for exact starts."""
    base = spec.initial_point()
    q0 = np.empty((chains, spec.n))
    for c in range(chains):
        iv = None
        if initvals is not None:
            iv = initvals[c] if isinstance(initvals, (list, tuple)) else initvals
        if isinstance(iv, np.ndarray):  # an explicit raveled start point is used as given (no jitter): parity tests pass these
            q0[c] = iv
            continue
        start = base.copy()
        if isinstance(iv, dict):
            for v in spec.vars:
                if v.name in iv:
                    start[v.offset : v.offset + v.size] = np.ravel(iv[v.name])
        g = np.random.default_rng(jitter_seeds[c])
        q = start
        for _ in range(jitter_max_retries + 1):
            q = start + g.uniform(-1.0, 1.0, spec.n) if jitter else start
            if logp_fn is None:
                break
            if np.isfinite(logp_fn(q[None])[0][0]):
                break
            if not jitter:
                raise SamplingError(f"Initial evaluation of model at starting point failed for chain {c}: logp is not finite")
        else:  # _init_jitter raises after jitter_max_retries (pymc/sampling/mcmc.py:1744-1754)
            raise SamplingError(f"no finite-logp jittered start found for chain {c} after {jitter_max_retries} retries")
        q0[c] = q
    return q0


def map_and_neg_hessian(cm, start, maxeval: int = 5000, rel_step: float = 1e-5):
    """init="map" (sampling/mcmc.py:1981-1985): ``start = find_MAP()``; ``cov = -find_hessian(start, negate_output=False)``.

    ``find_MAP`` (tuning/starting.py:52-190) minimises ``-logp`` over the unconstrained vector with SciPy's L-BFGS-B using the
    model's own logp/dlogp, from the initial point, with at most ``maxeval`` evaluations: the same call here, on the engine's
    ``logp_dlogp``.  The Hessian the reference compiles symbolically (``Model.compile_d2logp``) is taken as central differences
    of the gradient -- all 2n displaced points in ONE batched device call.  The reference hands ``-H`` to ``QuadPotentialFull``
    as its covariance, and so does this (the docstring of find_MAP advises against this initialisation; it is here for parity of
    the ``init`` surface).  Returns (q_map[n], cov[n, n])."""
    from scipy import optimize

    start = np.asarray(start, dtype=np.float64)
    n = start.size

    def cost(x):
        lp, g = cm.logp_dlogp(x[None, :])
        return -float(lp[0]), -np.asarray(g[0], dtype=np.float64)

    res = optimize.minimize(cost, start, jac=True, method="L-BFGS-B", options={"maxfun": int(maxeval)})
    q = np.asarray(res.x, dtype=np.float64)
    h = rel_step * np.maximum(1.0, np.abs(q))
    pts = np.concatenate([q[None, :] + np.diag(h), q[None, :] - np.diag(h)])
    _, g = cm.logp_dlogp(pts)
    H = (np.asarray(g[:n]) - np.asarray(g[n:])) / (2.0 * h)[:, None]
    H = 0.5 * (H + H.T)
    return q, -H


def sample_b200_nuts(
    draws: int = 1000,
    *,
    tune: int = 1000,
    chains: int = 4,
    target_accept: float | None = None,
    random_seed=None,
    initvals=None,
    jitter: bool = True,
    model: ModelSpec | ModelIR | CompiledModel | None = None,
    var_names=None,
    nuts_kwargs: dict | None = None,
    progressbar: bool = False,
    quiet: bool = True,
    keep_untransformed: bool = False,
    chain_method: str = "vectorized",
    idata_kwargs: dict | None = None,
    compute_convergence_checks: bool = True,
    discard_tuned_samples: bool = True,
    momentum: str = "device",
    nuts_sampler: str = "b200",
    init: str = "auto",
    step: str = "nuts",
    gather: str = "rank0",
) -> SampleResult:
    """Draw samples from the posterior using the CUDA engine.

    Arguments follow ``sample_jax_nuts`` (pymc/sampling/jax.py:495-517).  ``model``: a ``pymc_b200.ir.ModelIR`` (any model
    of the closed factor set; ``from_pymc`` lowers a ``pm.Model`` to one), a ``ModelSpec`` naming a hand-written kernel, or
    a ``CompiledModel``.  ``nuts_kwargs`` accepts the ``pm.NUTS`` / ``pm.HamiltonianMC`` keywords ``max_treedepth,
    early_max_treedepth, step_scale, gamma, k, t0, Emax, adapt_step_size, path_length, max_steps`` and ``potential`` (one of the
    reference's ``QuadPotential*`` objects: read and mapped onto the engine's mass kinds, ``pymc_b200.potentials``).
    ``init`` (pm.sample / init_nuts, pymc/sampling/mcmc.py:1759-2021): "auto" = "jitter+adapt_diag"; "adapt_diag";
    "jitter+adapt_diag_grad" (QuadPotentialDiagAdaptExp, alpha 0.02, stop at tune - 50 when tune > 250);
    "adapt_full" / "jitter+adapt_full" (QuadPotentialFullAdapt: a dense covariance per chain, identity start, weight 10,
    mcmc.py:1986-2005); "map" (every chain starts at the L-BFGS-B optimum, QuadPotentialFull(-Hessian), mcmc.py:1981-1985);
    "advi", "advi+adapt_diag", "advi_map" (mean-field ADVI on the engine's logp/dlogp, ``pymc_b200.advi``; ``nuts_kwargs["n_init"]``
    caps its iterations, default 200000, mcmc.py:1913-1980).
    ``step``: "nuts" (target_accept default 0.8) or "hmc" (HamiltonianMC, default 0.65).
    ``momentum="numpy"`` draws the momentum normals from each chain's NumPy potential stream exactly like
    the reference (host-generated, uploaded); ``"device"`` generates them on the GPU (Philox).
    Multi-GPU (torch.distributed initialised, one process per GPU): chains are sharded over the ranks; ``gather="rank0"``
    collects all chains on rank 0 (the other ranks return their own shard, ``attrs["chains_held"]`` says which),
    ``"all"`` gives every rank everything (world-size times the traffic), ``"none"`` leaves the posterior sharded.
    ``idata_kwargs={"log_likelihood": True}`` adds the pointwise log-likelihood group (IR models; evaluated on the device).
    Posterior values are constrained ON THE DEVICE where each draw is recorded (the backward transform is fused into the
    kernel); ``keep_untransformed=True`` records the unconstrained positions and transforms on the host instead.
    """
    if model is None:
        raise TypeError("model is required (a pymc_b200.ir.ModelIR, a pymc_b200.models.ModelSpec or a CompiledModel)")
    if chain_method not in ("vectorized", "parallel"):
        raise ValueError("chain_method must be 'vectorized' or 'parallel'")
    if step not in ("nuts", "hmc"):
        raise ValueError("step must be 'nuts' or 'hmc'")
    cm = model if hasattr(model, "nuts_run") else CompiledModel(model)  # a CompiledModel (or an object with its interface)
    spec = cm.spec
    nk = dict(nuts_kwargs or {})
    if target_accept is None:
        target_accept = 0.8 if step == "nuts" else 0.65  # base_hmc.py:91 / hmc.py:142
    nk.setdefault("target_accept", target_accept)
    if step == "hmc":
        nk["sampler"] = "hmc"
    if init == "auto":
        init = "jitter+adapt_diag"
    if init.startswith("jitter+"):
        init = init[len("jitter+"):]
    else:
        jitter = False
    if init == "adapt_diag":
        mass = "diag_adapt"
    elif init == "adapt_diag_grad":
        mass = "diag_adapt_grad"
        nk.setdefault("mass_alpha", 0.02)
        nk.setdefault("stop_adaptation", tune - 50 if tune > 250 else None)  # mcmc.py:1900-1903
    elif init == "adapt_full":
        mass = "dense_adapt"  # QuadPotentialFullAdapt(n, mean, eye, 10): mcmc.py:1986-2005
    elif init == "map":
        mass = "dense"        # every chain starts at the MAP; QuadPotentialFull(-Hessian): mcmc.py:1981-1985 (resolved below)
    elif init in ("advi", "advi_map"):
        mass = "diag"         # QuadPotentialDiag(approx.std**2), start points drawn from the approximation: mcmc.py:1940-1980
    elif init == "advi+adapt_diag":
        mass = "diag_adapt"   # QuadPotentialDiagAdapt(n, approx.mean, approx.std**2, 50): mcmc.py:1913-1938
    else:
        raise ValueError(f"init={init!r}: implemented initialisations are (jitter+)adapt_diag, (jitter+)adapt_diag_grad, "
                         "(jitter+)adapt_full, map, advi, advi+adapt_diag and advi_map")
    mass = nk.pop("mass", mass)  # "dense": QuadPotentialFull with the model's covariance (MvNormal models)
    # pm.NUTS(potential=...) (hmc/base_hmc.py:82-169): a reference QuadPotential object replaces init's mass matrix
    pot_var0 = pot_mean0 = None
    potential = nk.pop("potential", None)
    if potential is not None:
        from . import potentials

        pk = potentials.engine_kwargs(potential, spec.n)
        mass = pk.pop("mass")
        pot_var0, pot_mean0 = pk.pop("var0", None), pk.pop("mean0", None)
        if "dense_cov" in pk:
            cm.set_dense_mass(cov=pk.pop("dense_cov"))
        elif "dense_inverse" in pk:
            cm.set_dense_mass(inverse=pk.pop("dense_inverse"))
        for k_, v_ in pk.items():
            if k_ in nk and nk[k_] != v_:
                raise ValueError(f"nuts_kwargs[{k_!r}] contradicts the potential object ({nk[k_]!r} vs {v_!r})")
            nk[k_] = v_

    from . import parallel

    lo, hi = parallel.my_chain_range(chains)
    step_rngs, pot_rngs, jitter_seeds = brng.chain_generators(random_seed, chains)
    q0_all = initial_points(spec, chains, jitter_seeds, initvals, jitter, cm.logp_dlogp)
    if init == "map" and potential is None:
        q_map, cov = map_and_neg_hessian(cm, q0_all[0])
        q0_all = np.broadcast_to(q_map, q0_all.shape).copy()  # initial_points = [start] * chains
        cm.set_dense_mass(cov=cov)
    advi_mean = None
    if init.startswith("advi") and potential is None:
        from . import advi

        start = map_and_neg_hessian(cm, q0_all[0])[0] if init == "advi_map" else q0_all[0]  # MeanField(start=find_MAP())
        seeds = np.random.SeedSequence(random_seed).spawn(2) if not isinstance(random_seed, np.random.Generator) else [random_seed] * 2
        advi_mean, advi_std, advi_it = advi.fit_meanfield(cm.logp_dlogp, start, n=int(nk.pop("n_init", 200_000)), seed=seeds[0])
        g = np.random.default_rng(seeds[1])
        q0_all = advi_mean + advi_std * g.standard_normal((chains, spec.n))  # approx.sample(draws=chains)
        pot_var0 = advi_std**2
        if init == "advi+adapt_diag":
            pot_mean0 = advi_mean
            nk.setdefault("mass_initial_weight", 50.0)
    # init_nuts: mean start point over ALL chains as the estimator's prior mean (mcmc.py:1890-1894)
    mean0 = np.broadcast_to(q0_all.mean(axis=0) if pot_mean0 is None else pot_mean0, (hi - lo, spec.n)).copy()
    if pot_var0 is not None:
        nk["var0"] = np.broadcast_to(pot_var0, (hi - lo, spec.n)).copy()
    states = brng.pack_pcg64(step_rngs[lo:hi])
    z = brng.momentum_noise(pot_rngs[lo:hi], tune + draws, spec.n) if momentum == "numpy" else None
    # Philox key of the device momentum noise: an independent child of the root seed (never a function of a chain's jitter)
    seed_key = brng.philox_key(random_seed) if z is None else 0
    # draws recorded in constrained space by the kernel itself (engines that implement `constrain`; test stand-ins do not)
    want_ll = bool((idata_kwargs or {}).get("log_likelihood", False))  # needs the unconstrained draws on the host
    on_device = (not keep_untransformed) and getattr(cm, "supports_constrain", False) and not want_ll
    if on_device:
        nk["constrain"] = True

    t0 = time.perf_counter()
    res = cm.nuts_run(q0_all[lo:hi], states, tune=tune, draws=draws, mean0=mean0, z=z, philox_seed=seed_key,
                      store_warmup=not discard_tuned_samples, mass=mass, chain_offset=lo, **nk)
    sampling_time = time.perf_counter() - t0
    bad = res.summary["bad_energy_at"]
    if np.any(bad >= 0):
        c = int(np.argmax(bad >= 0))
        raise SamplingError(f"Bad initial energy in chain {lo + c} at iteration {int(bad[c])}: check any log "
                            "probabilities that are inf or nan (model.debug())")
    d_all, st_all = res.draws, res.stats
    held = (lo, hi)
    if parallel.world_size() > 1 and gather != "none":
        if gather not in ("rank0", "all"):
            raise ValueError("gather must be 'rank0', 'all' or 'none'")
        g_d, g_st = parallel.gather_chains(d_all, st_all, chains, dst=None if gather == "all" else 0)
        if g_d is not None:
            d_all, st_all, held = g_d, g_st, (0, chains)

    w = tune if not discard_tuned_samples else 0

    def pack(dq, st):
        post = spec.split_rv(dq) if on_device else spec.constrain(dq)
        ir_ = getattr(cm, "ir", None)
        if ir_ is not None and getattr(ir_, "deterministics", None):  # pm.Deterministic values, from the constrained draws
            post.update(ir_.eval_deterministics(post))
        if var_names is not None:
            post = {k: v for k, v in post.items() if k in var_names}
        stats = {_STAT_RENAME[k]: (v.astype(bool) if v.dtype == np.uint8 else v) for k, v in st.items()}
        return post, stats

    post, stats = pack(d_all[:, w:], {k: v[:, w:] for k, v in st_all.items()})
    out = SampleResult(post, stats, d_all[:, w:] if keep_untransformed else None)
    ir = getattr(cm, "ir", None)
    if ir is not None:
        out.observed_data, out.constant_data = ir.observed_data(), ir.constant_data()
    elif getattr(spec, "data", None):
        obs = {"y"}
        out.observed_data = {k: np.asarray(v) for k, v in spec.data.items() if k in obs}
        out.constant_data = {k: np.asarray(v) for k, v in spec.data.items() if k not in obs and np.ndim(v) == 1}
    if want_ll:
        out.log_likelihood = _log_likelihood(cm, d_all[:, w:])
    if w:
        out.warmup_posterior, out.warmup_sample_stats = pack(d_all[:, :w], {k: v[:, :w] for k, v in st_all.items()})
    out.attrs = {"sampling_time": sampling_time, "tuning_steps": tune, "inference_library": "pymc_b200", "chains_held": held,
                 "kernel_ms": res.kernel_ms, "grad_evals": int(st_all["tree_size"].sum())}
    if compute_convergence_checks and d_all.shape[0] > 1 and draws >= 8:
        from . import diagnostics

        out.attrs["ess_bulk_min"], out.attrs["rhat_max"] = diagnostics.convergence_summary(d_all[:, w:])
        out.attrs["divergences"] = int(stats["diverging"].sum())
    return out
