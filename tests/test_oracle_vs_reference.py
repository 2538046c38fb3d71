"""CPU: oracle/nuts_numpy.py must be BIT-IDENTICAL to the reference's own nuts.py / integration.py / quadpotential.py /
step_sizes.py.  The reference chains were produced by those files loaded verbatim (oracle/ref_loader.py) and are stored in
tests/golden/reference_chains.npz (oracle/make_reference_chains.py)."""
import numpy as np
import pytest

from oracle import logp_numpy, nuts_numpy
from oracle.make_reference_chains import DENSE_ADAPT_STATS, PORT_CASES, PORT_STATS, port_key
from pymc_b200 import models


@pytest.fixture(scope="module")
def ref(golden):
    return golden("reference_chains")


def _port_chain(spec, f, q0, seed, tune, draws, adapt):
    mass = nuts_numpy.DiagMass(np.ones(spec.n), adapt=adapt, initial_mean=q0.copy(), initial_weight=10)
    o = nuts_numpy.Oracle(f, mass, adapt_step_size=adapt)
    o.setup_chain(np.random.default_rng(seed))
    if tune == 0:
        o.tune = False
    return o.run(q0, tune, draws)


@pytest.mark.parametrize("name,adapt,tune,draws", PORT_CASES)
def test_port_is_bit_identical_to_reference(ref, name, adapt, tune, draws):
    spec = models.std_normal(40) if name == "std_normal" else models.BUILDERS[name]()
    f = logp_numpy.make_logp(spec)
    q0 = spec.initial_point() + np.random.default_rng(1).uniform(-1, 1, spec.n)
    qo, so = _port_chain(spec, f, q0, 77, tune, draws, adapt)
    key = port_key(name, adapt, tune, draws)
    assert np.array_equal(ref[key + "_q"], qo)
    for k in PORT_STATS:
        assert np.array_equal(ref[f"{key}_{k}"], so[k]), k


def test_dense_mass_matches_reference(ref):
    """QuadPotentialFull (quadpotential.py:680-725) vs DenseMass, fixed step size."""
    spec = models.mvgauss(n=15, seed=2)
    f = logp_numpy.make_logp(spec)
    q0 = np.random.default_rng(3).normal(size=15)
    o = nuts_numpy.Oracle(f, nuts_numpy.DenseMass(spec.data["cov"]), adapt_step_size=False)
    o.setup_chain(np.random.default_rng(5))
    o.tune = False
    qo, _ = o.run(q0, 0, 12)
    assert np.array_equal(ref["dense_full_q"], qo)


@pytest.mark.parametrize("name,tune,draws", [("eight_schools", 130, 10), ("radon", 60, 5)])
def test_dense_adapt_mass_matches_reference(ref, name, tune, draws):
    """QuadPotentialFullAdapt (quadpotential.py:748-845, init="adapt_full": mcmc.py:1986-1996) vs DenseAdaptMass, through the
    first window switch for Eight Schools (foreground <- background at delta = 101)."""
    spec = models.BUILDERS[name]()
    n = spec.n
    f = logp_numpy.make_logp(spec)
    q0 = spec.initial_point() + np.random.default_rng(4).uniform(-1, 1, n)
    o = nuts_numpy.Oracle(f, nuts_numpy.DenseAdaptMass(n, q0.copy(), np.eye(n), 10))
    o.setup_chain(np.random.default_rng(91))
    qo, so = o.run(q0, tune, draws)
    key = f"dense_adapt_{name}"
    assert np.array_equal(ref[key + "_q"], qo)
    for k in DENSE_ADAPT_STATS:
        assert np.array_equal(ref[f"{key}_{k}"], so[k]), k
    assert np.array_equal(ref[key + "_cov"], o.mass.cov) and np.array_equal(ref[key + "_chol"], o.mass.chol)


def test_loader_self_check_known_answer():
    """The known answer of the reference loader's self-check (SURVEY 8c): five Eight-Schools draws the verbatim reference
    produced (depth, tree_size, index_in_trajectory, energy, positions), reproduced by the NumPy port."""
    spec = models.eight_schools()
    f = logp_numpy.make_logp(spec)
    qo, so = _port_chain(spec, f, np.zeros(10), 20240922, 0, 5, False)
    got = [(int(d), int(t), int(i)) for d, t, i in zip(so["depth"], so["tree_size"], so["index_in_trajectory"])]
    assert got == [(4, 15, -10), (5, 31, -10), (5, 31, -11), (5, 31, 13), (4, 15, 10)]
    assert abs(so["energy"][0] - 48.33000583528482) < 1e-10
    assert abs(qo[0][0] - (-0.4558081288677123)) < 1e-12 and abs(qo[0][1] - 2.267682240205048) < 1e-12
