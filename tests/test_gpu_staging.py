"""-m gpu: the memory modes of the C ABI give the same bits.  Host arrays are staged through the model's device arena (or
their own buffers, or written through the UVA alias of page-locked memory); device arrays are used in place."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _model():
    from pymc_b200 import engine, ir

    m = ir.radon_ir(60, 5, 3)
    return m, engine.CompiledModel(m, specialise=False)


def _inputs(m, C, T, seed=3):
    from pymc_b200 import rng as brng

    sr, pr, _ = brng.chain_generators(seed, C)
    q0 = m.initial_point() + np.random.default_rng(seed).uniform(-0.3, 0.3, (C, m.n))
    z = brng.momentum_noise(pr, T, m.n)
    return q0, brng.pack_pcg64(sr), z


def _host(res):
    """(draws, stats, summary) of a NutsResult as fresh NumPy arrays (pinned pools are reused, CUDA tensors copied back)."""
    to_np = lambda a: a.cpu().numpy() if hasattr(a, "cpu") else np.array(a)  # noqa: E731
    return to_np(res.draws), {k: to_np(v) for k, v in res.stats.items()}, {k: to_np(v) for k, v in res.summary.items()}


def _assert_same(a, b):
    assert np.array_equal(a[0], b[0], equal_nan=True)
    for part in (1, 2):
        assert a[part].keys() == b[part].keys()
        for k in a[part]:
            assert np.array_equal(a[part][k], b[part][k], equal_nan=True), k


TUNE, DRAWS = 20, 20
RUN_KW = dict(tune=TUNE, draws=DRAWS, mass="diag", adapt_step_size=False, philox_seed=4)


def test_nuts_run_outputs_are_identical_in_host_pinned_and_device_memory():
    from pymc_b200 import _lib

    m, cm = _model()
    C = 12
    q0, rng0, z = _inputs(m, C, TUNE + DRAWS)
    kw = dict(RUN_KW, var0=np.full((C, m.n), 0.9), mean0=q0, eps0=np.full(C, 0.05), z=z)
    out, rngs = [], []
    for mode in ({}, {"pinned_outputs": True}, {"device_outputs": True}):
        rng = rng0.copy()
        out.append(_host(cm.nuts_run(q0, rng, **kw, **mode)))
        rngs.append(rng)
    assert out[0][1].keys() == {name for name, _ in _lib.STAT_FIELDS}
    for o, r in zip(out[1:], rngs[1:]):
        _assert_same(o, out[0])
        assert np.array_equal(r, rngs[0])
    assert not np.array_equal(rngs[0], rng0)  # the step streams advanced


def test_a_split_run_through_a_grown_staging_arena_is_identical_to_the_whole_run():
    from pymc_b200 import engine

    m, cm = _model()
    C, T = 6, TUNE + DRAWS
    q0, rng0, z = _inputs(m, C, T)
    kw = dict(RUN_KW, var0=np.full((C, m.n), 0.9), eps0=np.full(C, 0.05))
    rng = rng0.copy()
    whole = _host(cm.nuts_run(q0, rng, z=z, **kw))

    # a second handle whose staging arena a larger run (more chains, chain state in and out) has grown first
    _, grown = _model()
    Cb = 3 * C
    qb, rb, zb = _inputs(m, Cb, T, seed=8)
    sb = engine.ChainState(Cb, m.n)
    grown.nuts_run(qb, rb, z=zb[:, :17], iter_count=17, save=sb, **RUN_KW)
    grown.nuts_run(qb, rb, z=zb[:, 17:], iter_begin=17, resume=sb, save=engine.ChainState(Cb, m.n), **RUN_KW)

    cut = 13  # inside the tuning phase
    rs = rng0.copy()
    s1, s2 = engine.ChainState(C, m.n), engine.ChainState(C, m.n)
    a = _host(cm.nuts_run(q0, rs, z=z[:, :cut], iter_count=cut, save=s1, **kw))
    b = _host(grown.nuts_run(q0, rs, z=z[:, cut:], iter_begin=cut, resume=s1, save=s2, **kw))
    joined = (np.concatenate([a[0], b[0]], axis=1), {k: np.concatenate([a[1][k], b[1][k]], axis=1) for k in a[1]}, b[2])
    _assert_same(joined, whole)
    assert np.array_equal(rs, rng)
    assert np.array_equal(s2.q, whole[0][:, -1])


def test_logp_leapfrog_and_pointwise_loglik_are_identical_for_host_and_device_arrays():
    import torch

    from pymc_b200 import _lib

    m, cm = _model()
    lib, h = cm._lib, cm._h
    Cn, n = 7, m.n
    rs = np.random.default_rng(5)
    q = m.initial_point() + rs.uniform(-0.5, 0.5, (Cn, n))
    dev = lambda a: torch.as_tensor(a, device="cuda").contiguous()  # noqa: E731
    back = lambda t: t.cpu().numpy()  # noqa: E731

    lp, g = np.empty(Cn), np.empty((Cn, n))
    _lib.check(lib.b200_logp_dlogp(h, q.ctypes.data, Cn, lp.ctypes.data, g.ctypes.data, _lib.MEM_HOST, None))
    qd, lpd, gd = dev(q), torch.empty(Cn, dtype=torch.float64, device="cuda"), torch.empty((Cn, n), dtype=torch.float64, device="cuda")
    _lib.check(lib.b200_logp_dlogp(h, qd.data_ptr(), Cn, lpd.data_ptr(), gd.data_ptr(), _lib.MEM_DEVICE, None))
    torch.cuda.synchronize()
    assert np.array_equal(back(lpd), lp) and np.array_equal(back(gd), g)

    var, eps = rs.uniform(0.5, 1.5, (Cn, n)), np.full(Cn, 0.03)
    state = dict(q=q.copy(), p=rs.normal(size=(Cn, n)), v=np.zeros((Cn, n)), grad=g.copy(), energy=np.zeros(Cn), logp=lp.copy(),
                 idx=np.arange(Cn, dtype=np.int64))
    order = ["q", "p", "v", "grad", "energy", "logp", "idx"]
    hs = {k: v.copy() for k, v in state.items()}
    _lib.check(lib.b200_leapfrog(h, var.ctypes.data, eps.ctypes.data, 6, Cn, *(hs[k].ctypes.data for k in order), _lib.MEM_HOST, None))
    ds = {k: dev(v) for k, v in state.items()}
    vd, ed = dev(var), dev(eps)
    _lib.check(lib.b200_leapfrog(h, vd.data_ptr(), ed.data_ptr(), 6, Cn, *(ds[k].data_ptr() for k in order), _lib.MEM_DEVICE, None))
    torch.cuda.synchronize()
    assert not np.array_equal(hs["q"], state["q"])
    for k in order:
        assert np.array_equal(back(ds[k]), hs[k]), k

    D, N = 9, len(m.likelihoods[0].y)
    draws = m.initial_point() + rs.uniform(-0.5, 0.5, (D, n))
    ll = np.empty((D, N))
    _lib.check(lib.b200_pointwise_loglik(h, 0, draws.ctypes.data, D, ll.ctypes.data, _lib.MEM_HOST, None))
    dd, lld = dev(draws), torch.empty((D, N), dtype=torch.float64, device="cuda")
    _lib.check(lib.b200_pointwise_loglik(h, 0, dd.data_ptr(), D, lld.data_ptr(), _lib.MEM_DEVICE, None))
    torch.cuda.synchronize()
    assert np.array_equal(back(lld), ll)
