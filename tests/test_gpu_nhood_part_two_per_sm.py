"""GPU parity of the region replay over partitioned swap targets (shuffle_algo 9) in its two-CTAs-per-SM shape: 512-thread
CTAs, two resident per SM, with regions sized for half an SM's shared memory.  The list replay (algo 7, 1024 threads) is the
cross-check."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import NhoodPlan
from tools import synth

pytestmark = pytest.mark.gpu


def _permute(g, n_cls, base, st, algo, region=0, lib=None, n_libs=0, jgen_threads=None):
    plan = NhoodPlan(g.indptr, g.indices, n_cls)
    plan.set_option("shuffle_algo", algo)
    plan.set_option("shuffle_threads", 512 if algo == 9 else 1024)
    plan.set_option("shuffle_r", 2)
    plan.set_option("shuffle_region", region)
    if jgen_threads is not None:
        plan.set_option("jgen_threads", jgen_threads)
    if lib is None:
        plan.set_base(base)
    else:
        plan.set_base(base, lib, n_libs)
    out = plan.permute(st)
    tail = None
    if algo == 9:
        plan.upload(st)
        tail = plan.shuffled_labels(len(st) - 2, len(st))
    plan.close()
    return out, tail


def test_two_per_sm_equals_list_replay_full_size():
    """configs[1] shape (1M spots, 30 clusters): 13 regions per permutation; 300 permutations are more than two CTAs per SM
    of an H100, so the persistent loop wraps."""
    g = synth.hex_graph(1000, 1000)
    base = synth.categorical_labels(g.shape[0], 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
    st = spawn_states(3, 300)
    got, tail = _permute(g, 30, base, st, 9)
    np.testing.assert_array_equal(tail, ref.shuffle_labels(base, st[-2:]))
    exp, _ = _permute(g, 30, base, st, 7)
    np.testing.assert_array_equal(got, exp)


@pytest.mark.parametrize("region", [0, 160])
def test_two_per_sm_equals_list_replay_many_permutations_per_warp(region):
    """2500 permutations in segments of 2100 and 900 elements (see test_gpu_nhood_part_multiperm.py), replayed by 512-thread
    CTAs; region 160 gives 14 regions."""
    n, n_cls, P = 3000, 30, 2500
    g = sp.csr_matrix((np.ones(n - 1, np.float32), (np.arange(n - 1), np.arange(1, n))), shape=(n, n))
    base = (np.arange(n) * 13 % n_cls).astype(np.uint32)
    lib = np.zeros(n, np.int32)
    lib[2100:] = 1
    st = spawn_states(11 + region, P)
    got, tail = _permute(g, n_cls, base, st, 9, region, lib, 2, jgen_threads=32)
    np.testing.assert_array_equal(tail, ref.shuffle_labels(base, st[-2:], lib, 2))
    exp, _ = _permute(g, n_cls, base, st, 7, region, lib, 2, jgen_threads=32)
    np.testing.assert_array_equal(got, exp)
