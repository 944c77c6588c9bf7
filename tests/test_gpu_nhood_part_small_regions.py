"""GPU parity of the region replay over partitioned swap targets (shuffle_algo 9) at the configs[1] shape (1M spots, 30
clusters) with 16 regions of 62 512 positions, the most a segment may take.  Most slots then gather their tops from above
the region, over many windows, through the replay's one-window-ahead copies.  The list replay (algo 7) is the cross-check."""

from __future__ import annotations

import numpy as np
import pytest

from oracle import ref
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import NhoodPlan
from tools import synth

pytestmark = pytest.mark.gpu


def _permute(g, base, st, algo, threads):
    plan = NhoodPlan(g.indptr, g.indices, 30)
    plan.set_option("shuffle_algo", algo)
    plan.set_option("shuffle_threads", threads)
    plan.set_option("shuffle_r", 2)
    plan.set_option("shuffle_region", 62512)
    plan.set_base(base)
    out = plan.permute(st)
    tail = None
    if algo == 9:
        plan.upload(st)
        tail = plan.shuffled_labels(len(st) - 2, len(st))
    plan.close()
    return out, tail


@pytest.mark.parametrize("threads", [512, 1024])
def test_sixteen_regions_equal_list_replay_full_size(threads):
    """512 threads: two CTAs per SM (1024-slot windows); 1024 threads: one CTA per SM (2048-slot windows).  300 permutations
    are more than the persistent grid, so its loop wraps."""
    g = synth.hex_graph(1000, 1000)
    base = synth.categorical_labels(g.shape[0], 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
    st = spawn_states(5, 300)
    got, tail = _permute(g, base, st, 9, threads)
    np.testing.assert_array_equal(tail, ref.shuffle_labels(base, st[-2:]))
    exp, _ = _permute(g, base, st, 7, 1024)
    np.testing.assert_array_equal(got, exp)
