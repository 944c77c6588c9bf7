"""GPU parity tests of the region replay over partitioned swap targets (shuffle_algo 9, nhood_apply_part_kernel fed by
nhood_jgen_kernel<Q, true>): numpy-identical shuffles for any array length, region size, label width and library split."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import NhoodPlan
from tools import synth

pytestmark = pytest.mark.gpu


def _chain(n):
    return sp.csr_matrix((np.ones(n - 1, np.float32), (np.arange(n - 1), np.arange(1, n))), shape=(n, n))


def _check(n, n_cls, region, threads=1024, lib=None, n_libs=0, P=4, seed=0):
    g = _chain(n)
    base = (np.arange(n) * 13 % n_cls).astype(np.uint32)
    plan = NhoodPlan(g.indptr, g.indices, n_cls)
    plan.set_option("shuffle_algo", 9)
    plan.set_option("shuffle_threads", threads)
    plan.set_option("shuffle_region", region)
    if lib is None:
        plan.set_base(base)
    else:
        plan.set_base(base, lib, n_libs)
    st = spawn_states(seed + n + region, P)
    plan.upload(st)
    got = plan.shuffled_labels(0, P)
    plan.close()
    np.testing.assert_array_equal(got, ref.shuffle_labels(base, st, lib, n_libs) if lib is not None else ref.shuffle_labels(base, st))


# Region sizes with at most 16 regions per segment, so that algo 9 itself runs (larger arrays fall back to algo 7).
@pytest.mark.parametrize("region,ns", [(16, [2, 3, 17, 100, 255]), (48, [5, 200, 767]), (1000, [2049, 4099, 15999]),
                                       (30000, [70001, 200003]), (0, [2, 9, 2047, 2048, 2049, 70001, 200003])])
@pytest.mark.parametrize("threads", [1024, 512])
def test_partitioned_region_replay_u8(region, ns, threads):
    """Tiny regions put almost every step into another region than its top; lengths around the 2048-step block make windows
    straddle block edges; 0 = everything shared memory holds."""
    for n in ns:
        _check(n, 241, region, threads)


@pytest.mark.parametrize("region", [48, 1000, 30000, 0])
def test_partitioned_region_replay_u16_and_segments(region):
    """16-bit labels (more than 256 categories) and library segments of unequal length."""
    n = {48: 700, 1000: 14001, 30000: 200003, 0: 200003}[region]
    _check(n, 300, region)
    lib = (np.arange(n) * 7 % 3).astype(np.int32)
    lib[: n // 5] = 0  # unequal segments
    _check(n, 300, region, lib=lib, n_libs=3, P=2)
    _check(n, 241, region, lib=lib, n_libs=3, P=2)


def test_partitioned_region_replay_single_element_segments():
    """Segments of one element have no steps: their label is copied through (the label rows are not pre-filled)."""
    n = 5000
    lib = np.full(n, 1, np.int32)
    lib[0] = 0
    lib[-1] = 2
    _check(n, 50, 0, lib=lib, n_libs=3, P=3)


def test_partitioned_equals_list_replay_full_size():
    """configs[1] shape (1M spots, 30 clusters): the permutation counts of algo 9 equal those of the list replay (algo 7)."""
    g = synth.hex_graph(1000, 1000)
    base = synth.categorical_labels(g.shape[0], 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
    st = spawn_states(3, 300)
    out = {}
    for algo in (7, 9):
        plan = NhoodPlan(g.indptr, g.indices, 30)
        plan.set_option("shuffle_algo", algo)
        plan.set_option("shuffle_threads", 1024)
        plan.set_option("shuffle_r", 2)
        plan.set_base(base)
        out[algo] = plan.permute(st)
        if algo == 9:
            plan.upload(st)
            np.testing.assert_array_equal(plan.shuffled_labels(298, 300), ref.shuffle_labels(base, st[298:]))
        plan.close()
    np.testing.assert_array_equal(out[9], out[7])
