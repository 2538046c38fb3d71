"""Where the persistent NUTS kernel keeps the main tree of a draw (p_sum, proposal q, both edge states: 8 vectors per chain).

``NutsLaunch`` first picks the hot tree levels by the rule ``test_gpu_models.radon_hot_level`` replicates, then places the
main tree in shared memory when the CTA still fits with it, and in the chain's global scratch otherwise.  A CPU replica of
that rule is pinned against hand-worked thresholds, and Radon NUTS runs on both sides of the threshold are checked against
the oracle sampler.
"""
import numpy as np
import pytest

from test_gpu_models import (MAX_SMEM, _dominant_for_hot, _dominant_sizes, _nuts_against_oracle, npl_warp, nuts_warp_smem_bytes,
                             radon_data, radon_hot_level, radon_layout, radon_spec)

TREE_VECS = 8


def radon_tree_in_shared(shared, n, max_td=10):
    """NutsLaunch's placement of the main tree for a chain-per-warp model: True when the 8 chains of a CTA fit with their
    hot levels and their main trees in shared memory."""
    NP = 32 * npl_warp(n)
    hot = radon_hot_level(shared, n, max_td)
    assert hot is not None
    data = (shared + 15) & ~15
    return data + 8 * (nuts_warp_smem_bytes(NP, hot, 1) + TREE_VECS * NP * 8) <= MAX_SMEM


def _dominant_layout(d, J=85):
    return radon_layout(np.repeat(np.arange(J), _dominant_sizes(d, J)), J)


def test_tree_placement_replica_against_hand_worked_thresholds():
    """J = 85 (n = 175, NPL 6, NP = 192), hot 2: per chain 12768 B of q, g, hot levels and scalars plus 8 x 1536 B of tree,
    so the tree fits while the staged data takes at most 232448 - 8 x 25056 = 32000 B.  One dominant county of d, the other
    84 of 2 observations: rows round4(d), 4 and 4, K = round4(d) + 12, shared = 512 K + 4 (96 + 4).
      d = 48: K = 60, shared 31120 -> tree in shared memory
      d = 49: K = 64, shared 33168 -> tree in global memory (hot 2 still fits: 33168 + 8 x 12768 = 135312 B)"""
    assert nuts_warp_smem_bytes(192, 2, 1) + TREE_VECS * 192 * 8 == 25056
    for d, K, shared, tree in ((48, 60, 31120, True), (49, 64, 33168, False)):
        L = _dominant_layout(d)
        assert (L["K"], L["shared"]) == (K, shared), d
        assert radon_hot_level(shared, 175) == 2, d
        assert radon_tree_in_shared(shared, 175) == tree, d


def test_bench_layout_places_the_tree_in_shared_memory_and_large_layouts_do_not():
    from pymc_b200 import models

    spec = models.radon()  # the bench model: 919 observations in 85 counties
    J = spec.meta["n_counties"]
    L = radon_layout(spec.data["county_idx"], J)
    assert (L["K"], L["shared"]) == (44, 22928)
    assert radon_hot_level(L["shared"], spec.n) == 2 and radon_tree_in_shared(L["shared"], spec.n)
    # the layouts the sampler tests run with one hot level or none keep the tree in global memory
    for hot in (1, 0):
        shared = _dominant_layout(_dominant_for_hot(hot))["shared"]
        assert radon_hot_level(shared, 175) == hot and not radon_tree_in_shared(shared, 175)
    # NPL 8 (NP = 256): the tree alone is 8 x 16384 B per CTA on top of 8 x 16864 B, more than 227 KB with any data
    for J in (94, 125):
        assert npl_warp(2 * J + 5) == 8 and not radon_tree_in_shared(radon_layout(np.arange(J), J)["shared"], 2 * J + 5)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [48, 49], ids=["tree_shared", "tree_global"])
def test_radon_nuts_on_both_sides_of_the_tree_threshold(d):
    county, x, y = radon_data(_dominant_sizes(d), np.random.default_rng(d), extreme=False)
    assert radon_tree_in_shared(radon_layout(county, 85)["shared"], 175) == (d == 48)
    _nuts_against_oracle(radon_spec(county, x, y, 85), 0.02, f"tree_d{d}", T=12)
