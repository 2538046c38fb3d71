"""CPU: seam B2 inbound -- the reference's own QuadPotential objects are read and mapped onto the engine's mass kinds
(pymc_b200/potentials.py), and ``sample_b200_nuts(nuts_kwargs={"potential": obj})`` runs the chain that potential defines
(checked on the oracle-backed engine, which is bit-identical to the reference).  The mapping reads only an object's class
name and attributes, so the objects here are stand-ins carrying the instance state of the reference's own objects, stored
in tests/golden/reference_chains.npz (oracle/make_reference_chains.py)."""
import numpy as np
import pytest

from b200_helpers import OracleEngine
from pymc_b200 import models, potentials, sampling


@pytest.fixture(scope="module")
def pot(golden):
    """case -> a stand-in object with the class name and attributes of the reference object of that case."""
    ref = golden("reference_chains")
    classes = {}

    def make(case):
        prefix = f"pot_{case}__"
        name = str(ref[prefix + "class"])
        cls = classes.setdefault(name, type(name, (), {}))
        obj = cls()
        for key in ref:
            if key.startswith(prefix) and key != prefix + "class":
                val = ref[key]
                setattr(obj, key[len(prefix):], val.item() if val.ndim == 0 else val.copy())
        return obj

    return make


def test_reference_potential_objects_map_onto_the_engine_kinds(pot):
    # the constructor arguments of the stored objects (oracle/make_reference_chains.py: potential_cases)
    n = 4
    rng = np.random.default_rng(0)
    v, mean = rng.uniform(0.5, 2.0, n), rng.normal(size=n)
    k = potentials.engine_kwargs(pot("diag"), n)
    assert k["mass"] == "diag" and np.array_equal(k["var0"], v)
    k = potentials.engine_kwargs(pot("diag_adapt"), n)
    assert (k["mass"], k["mass_initial_weight"], k["adaptation_window"], k["discard_window"]) == ("diag_adapt", 7.0, 33, 9)
    assert np.array_equal(k["var0"], v) and np.array_equal(k["mean0"], mean)
    k = potentials.engine_kwargs(pot("diag_adapt_exp"), n)
    assert (k["mass"], k["mass_alpha"], k["stop_adaptation"], k["discard_window"]) == ("diag_adapt_grad", 0.03, 120, 50)
    assert potentials.engine_kwargs(pot("diag_adapt_exp_nostop"), n)["stop_adaptation"] is None
    B = rng.normal(size=(n, n))
    cov = B @ B.T + n * np.eye(n)
    k = potentials.engine_kwargs(pot("full"), n)
    assert k["mass"] == "dense" and np.array_equal(k["dense_cov"], cov)
    k = potentials.engine_kwargs(pot("full_inv"), n)
    assert k["mass"] == "dense" and np.allclose(k["dense_inverse"], cov, rtol=1e-13, atol=1e-13)
    k = potentials.engine_kwargs(pot("full_adapt"), n)
    assert (k["mass"], k["mass_initial_weight"], k["adaptation_window"], k["window_multiplier"], k["update_window"]) == \
           ("dense_adapt", 10.0, 40, 3.0, 5)
    assert np.array_equal(k["var0"], v) and np.array_equal(k["mean0"], mean)
    with pytest.raises(NotImplementedError, match="non-diagonal"):
        potentials.engine_kwargs(pot("full_adapt_nondiag"), n)
    # options the kernels do not implement are refused by name, never ignored
    with pytest.raises(NotImplementedError, match="early_update"):
        potentials.engine_kwargs(pot("diag_adapt_early"), n)
    with pytest.raises(NotImplementedError, match="multiplier"):
        potentials.engine_kwargs(pot("diag_adapt_multiplier"), n)
    with pytest.raises(NotImplementedError, match="use_grads"):
        potentials.engine_kwargs(pot("diag_adapt_exp_nograds"), n)

    class Mine(type(pot("diag"))):  # the user-subclass case of tests/step_methods/hmc/test_quadpotential.py:138-157
        def velocity(self, x, out=None):
            return x

    mine = Mine()
    mine.v = v
    with pytest.raises(NotImplementedError, match="subclass"):
        potentials.engine_kwargs(mine, n)
    with pytest.raises(ValueError, match="expected 4 values"):
        potentials.engine_kwargs(pot("diag_n3"), n)


def test_a_potential_object_defines_the_chain_the_sampler_runs(pot):
    """nuts_kwargs={"potential": QuadPotentialDiagAdapt(...)}: every chain equals the reference chain under that potential."""
    from oracle import logp_numpy, nuts_numpy
    from pymc_b200 import rng as brng

    spec = models.eight_schools()
    n, chains, seed, tune, draws = spec.n, 2, 6, 45, 8
    rng = np.random.default_rng(1)
    mean, diag = rng.normal(size=n), rng.uniform(0.5, 2.0, n)
    adapt = pot("es_diag_adapt")  # QuadPotentialDiagAdapt(n, mean, diag, 4, adaptation_window=20, discard_window=5)
    res = sampling.sample_b200_nuts(draws, tune=tune, chains=chains, random_seed=seed, model=OracleEngine(spec), momentum="numpy",
                                    keep_untransformed=True, nuts_kwargs={"potential": adapt})
    step_rngs, pot_rngs, jitter_seeds = brng.chain_generators(seed, chains)
    q0 = sampling.initial_points(spec, chains, jitter_seeds)
    f = logp_numpy.make_logp(spec)
    for c in range(chains):
        m = nuts_numpy.DiagMass(diag, adapt=True, initial_mean=mean.copy(), initial_weight=4, adaptation_window=20, discard_window=5)
        o = nuts_numpy.Oracle(f, m)
        o.rng, o.mass.rng = step_rngs[c], pot_rngs[c]
        qs, _ = o.run(q0[c], tune, draws)
        assert np.array_equal(qs[tune:], res.unconstrained[c])
    fixed = sampling.sample_b200_nuts(draws, tune=tune, chains=1, random_seed=seed, model=OracleEngine(spec), momentum="numpy",
                                      keep_untransformed=True, nuts_kwargs={"potential": pot("es_diag")})
    m = nuts_numpy.DiagMass(diag, adapt=False)
    o = nuts_numpy.Oracle(f, m)
    sr, pr, js = brng.chain_generators(seed, 1)
    o.rng, o.mass.rng = sr[0], pr[0]
    qs, _ = o.run(sampling.initial_points(spec, 1, js)[0], tune, draws)
    assert np.array_equal(qs[tune:], fixed.unconstrained[0])
    with pytest.raises(ValueError, match="contradicts"):
        sampling.sample_b200_nuts(2, tune=2, chains=1, random_seed=1, model=OracleEngine(spec), momentum="numpy",
                                  nuts_kwargs={"potential": adapt, "adaptation_window": 99})
