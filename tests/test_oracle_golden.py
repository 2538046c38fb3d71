"""CPU: oracle/nuts_numpy.py against the committed golden vectors (made by oracle/make_golden.py from the
reference's own code).  Fixed-step cases must reproduce whole chains; adaptive (chaotic) cases are
replayed draw by draw from the golden pre-draw state, which is robust to BLAS kernels of another CPU."""
import numpy as np
import pytest

from b200_helpers import SPEC_OF, TREE_KW
from oracle import logp_numpy, nuts_numpy


def _oracle(spec, f, var, adapt=False, dense=False, **kw):
    mass = nuts_numpy.DenseMass(spec.data["cov"]) if dense else nuts_numpy.DiagMass(var, adapt=adapt)
    return nuts_numpy.Oracle(f, mass, adapt_step_size=False, **kw)


def _gen_from_state(state_u64x4):
    g = np.random.default_rng(0)
    st = g.bit_generator.state
    st["state"]["state"] = (int(state_u64x4[0]) << 64) | int(state_u64x4[1])
    st["state"]["inc"] = (int(state_u64x4[2]) << 64) | int(state_u64x4[3])
    st["has_uint32"], st["uinteger"] = 0, 0
    g.bit_generator.state = st
    return g


@pytest.mark.parametrize("name", ["std_normal_fixed", "eight_schools_fixed", "radon_fixed", "std_normal_team_fixed",
                                  "stochvol_small_fixed", "stochvol_fixed", "logistic_small_fixed",
                                  "mvgauss_dense_fixed", "logistic_k128_fixed"])
def test_fixed_step_chains_reproduce_golden(golden, name):
    d = golden(name)
    spec = SPEC_OF[name]()
    f = logp_numpy.make_logp(spec)
    for c in range(len(d["seeds"])):
        o = _oracle(spec, f, d["var"][c], dense=bool(d["dense"]) if "dense" in d else False)
        o.da = nuts_numpy.DualAveraging(float(d["used_eps"][c][0]))
        o.rng, o.tune = _gen_from_state(d["pre_rng"][c][0]), False
        qs, st = o.run(d["q0"][c], 0, int(d["draws"]), z=d["z"][c])
        assert np.array_equal(st["tree_size"], d["stat_tree_size"][c])
        assert np.array_equal(st["index_in_trajectory"], d["stat_index_in_trajectory"][c])
        assert np.max(np.abs(qs - d["draws_q"][c])) <= 1e-9
        assert np.max(np.abs(st["energy"] - d["stat_energy"][c])) <= 1e-9


@pytest.mark.parametrize("name", ["eight_schools_adapt", "radon_small_adapt", "radon_adapt", "stochvol_small_adapt",
                                  "logistic_small_adapt"])
def test_single_draw_replay_of_adaptive_golden(golden, name):
    d = golden(name)
    spec = SPEC_OF[name]()
    f = logp_numpy.make_logp(spec)
    tune, T = int(d["tune"]), int(d["tune"]) + int(d["draws"])
    sel = range(0, T, 7 if name == "radon_adapt" else 3)
    q_prev = np.concatenate([d["q0"][0][None], d["draws_q"][0][:-1]])
    bad = 0
    for t in sel:
        o = _oracle(spec, f, d["pre_var"][0][t], **TREE_KW.get(name, {}))
        o.da = nuts_numpy.DualAveraging(float(d["used_eps"][0][t]))
        o.rng = _gen_from_state(d["pre_rng"][0][t])
        o.tune = t < tune
        o.iter_count = t
        o.adapt_step_size = False
        # the step size of a tuning draw is exp(log_step); with adaptation off current() reads log_bar == log_step here
        q, st = o.draw(q_prev[t], z=d["z"][0][t])
        same = (st["tree_size"] == d["stat_tree_size"][0][t]) and (st["depth"] == d["stat_depth"][0][t])
        if not same:
            bad += 1
            continue
        assert np.max(np.abs(q - d["draws_q"][0][t])) <= 1e-6
        assert st["diverging"] == bool(d["stat_diverging"][0][t])
    assert bad <= max(1, len(sel) // 50)


@pytest.mark.parametrize("name", ["eight_schools_warm_adapt", "radon_warm_adapt"])
def test_adaptation_prefix_reproduces_golden(golden, name):
    """Dual averaging + Welford bookkeeping: first 120 iterations (covers discard window and first switch)."""
    d = golden(name)
    spec = SPEC_OF[name]()
    f = logp_numpy.make_logp(spec)
    mass = nuts_numpy.DiagMass(d["init_var"][0], adapt=True, initial_mean=d["q0"][0].copy(), initial_weight=10)
    o = nuts_numpy.Oracle(f, mass, step_scale=float(d["step_scale"]))
    o.rng = _gen_from_state(d["pre_rng"][0][0])
    T = 120
    qs, st = o.run(d["q0"][0], T, 0, z=d["z"][0][:T])
    assert np.array_equal(st["tree_size"], d["stat_tree_size"][0][:T])
    assert np.max(np.abs(st["step_size"] - d["stat_step_size"][0][:T]) / d["stat_step_size"][0][:T]) <= 1e-9
    assert np.max(np.abs(qs - d["draws_q"][0][:T])) <= 1e-7


def test_dense_mass_step_adaptation_prefix_reproduces_golden(golden):
    """QuadPotentialFull (fixed dense covariance) + dual averaging: the first iterations of the reference run."""
    name = "mvgauss_dense_stepadapt"
    d = golden(name)
    spec = SPEC_OF[name]()
    f = logp_numpy.make_logp(spec)
    o = nuts_numpy.Oracle(f, nuts_numpy.DenseMass(spec.data["cov"]))
    o.rng = _gen_from_state(d["pre_rng"][0][0])
    T = 40
    qs, st = o.run(d["q0"][0], T, 0, z=d["z"][0][:T])
    assert np.array_equal(st["tree_size"], d["stat_tree_size"][0][:T])
    assert np.max(np.abs(st["step_size"] - d["stat_step_size"][0][:T]) / d["stat_step_size"][0][:T]) <= 1e-9
    assert np.max(np.abs(qs - d["draws_q"][0][:T])) <= 1e-7


def test_ms_weight_candidate_takes_the_reference_decisions(golden, monkeypatch):
    """The (m, s) multinomial-weight arithmetic of the persistent CUDA kernel (nuts_warp.cuh: log-weight = m + log s, one
    exp and no log per merge) restated here on top of the oracle: it must take exactly the decisions of the reference's
    logaddexp arithmetic on the golden chains."""
    import math

    class MSTrajectory(nuts_numpy._Trajectory):
        def __init__(self, *a):
            super().__init__(*a)
            self.s = 1.0

        def _leaf(self, frm, eps):
            span, div, turn = super()._leaf(frm, eps)
            span.s = 1.0
            return span, div, turn

        @staticmethod
        def _split(m2, s2, m1, s1):  # -> (w1, w2, m): weights of tree1 / tree2 relative to the larger m
            dm = m2 - m1
            e = math.exp(-abs(dm))
            return (s1 * e, s2, max(m1, m2)) if dm >= 0.0 else (s1, s2 * e, max(m1, m2))

        def _grow(self, frm, height, eps):
            if height == 0:
                return self._leaf(frm, eps)
            a, div, turn = self._grow(frm, height - 1, eps)
            if div or turn:
                return a, div, turn
            b, div, turn = self._grow(a.right, height - 1, eps)
            if not (div or turn):
                ps = a.p_sum + b.p_sum
                turn = nuts_numpy._uturn(ps, a.left.v, b.right.v)
                if (not turn) and (height - 1 > 0):
                    s1 = a.p_sum + b.left.p
                    turn = nuts_numpy._uturn(s1, a.left.v, b.left.v)
                    if not turn:
                        s2 = a.right.p + b.p_sum
                        turn = nuts_numpy._uturn(s2, a.right.v, b.right.v)
                w1, w2, m = self._split(b.log_w, b.s, a.log_w, a.s)
                ws = w1 + w2
                pick = b.pick if self.rng.random() * ws < w2 else a.pick
                out = nuts_numpy.Span(a.left, b.right, ps, pick, m)
                out.s = ws
                return out, div, turn
            out = nuts_numpy.Span(a.left, b.right, a.p_sum, a.pick, a.log_w)
            out.s = a.s
            return out, div, turn

        def double(self, direction):
            # the log-domain parent consumes rng and updates log_w; redo its bookkeeping with (m, s)
            if direction > 0:
                sub, div, turn = self._grow(self.right, self.depth, np.asarray(self.eps, dtype="float64"))
                lo_begin, lo_end, hi_begin, hi_end = self.left, self.right, sub.left, sub.right
                lo_sum, hi_sum = self.p_sum.copy(), sub.p_sum
                self.right = sub.right
            else:
                sub, div, turn = self._grow(self.left, self.depth, np.asarray(-self.eps, dtype="float64"))
                lo_begin, lo_end, hi_begin, hi_end = sub.right, sub.left, self.left, self.right
                lo_sum, hi_sum = sub.p_sum, self.p_sum.copy()
                self.left = sub.right
            self.depth += 1
            if div or turn:
                return div, turn
            wo, wn, m = self._split(sub.log_w, sub.s, self.log_w, self.s)
            if self.rng.random() * wo < wn:
                self.pick = sub.pick
            self.log_w, self.s = m, wo + wn
            self.p_sum[:] += sub.p_sum
            turn = nuts_numpy._uturn(self.p_sum, self.left.v, self.right.v)
            if not turn:
                turn = nuts_numpy._uturn(lo_sum + hi_begin.p, lo_begin.v, hi_begin.v)
            if not turn:
                turn = nuts_numpy._uturn(lo_end.p + hi_sum, lo_end.v, hi_end.v)
            return div, turn

    monkeypatch.setattr(nuts_numpy, "_Trajectory", MSTrajectory)
    for name in ("eight_schools_fixed", "radon_fixed", "stochvol_small_fixed"):
        d = golden(name)
        spec = SPEC_OF[name]()
        f = logp_numpy.make_logp(spec)
        for c in range(len(d["seeds"])):
            o = _oracle(spec, f, d["var"][c])
            o.da = nuts_numpy.DualAveraging(float(d["used_eps"][c][0]))
            o.rng, o.tune = _gen_from_state(d["pre_rng"][c][0]), False
            qs, st = o.run(d["q0"][c], 0, int(d["draws"]), z=d["z"][c])
            assert np.array_equal(st["tree_size"], d["stat_tree_size"][c])
            assert np.array_equal(st["index_in_trajectory"], d["stat_index_in_trajectory"][c])
            assert np.max(np.abs(qs - d["draws_q"][c])) <= 1e-9
