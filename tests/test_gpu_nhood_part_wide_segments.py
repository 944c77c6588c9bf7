"""GPU parity of the region replay over partitioned swap targets (shuffle_algo 9) on segments that only fit it with 32-bit
window tables, up to 32 regions per segment and more 2048-step blocks than threads: two 512-thread CTAs per SM.  The list
replay (algo 7, 1024 threads) is the cross-check.  Every case first restates the host's region cap (part_region_cap in
squidpy_b200/csrc/nhood.cu) to assert that it lands on the intended side of the shape rule."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import NhoodPlan
from tests import device_attrs
from tools import synth

pytestmark = pytest.mark.gpu

L = 2048  # SQB_PART_L
RMAX = 32  # SQB_PART_RMAX
NT = 512
_ATTR_SMEM_PER_SM = 81  # cudaDevAttrMaxSharedMemoryPerMultiprocessor
_ATTR_SMEM_RESERVED = 111  # cudaDevAttrReservedSharedMemoryPerBlock


def _regions(seg_lens, lt_bytes, region=0):
    """(regions of the most-cut segment, step blocks of the longest segment) of the two-per-SM shape."""
    nbmax = max((m + L - 1) // L for m in seg_lens)
    HS = 2 * NT
    tables = 2 * HS * 4 + 2 * HS * 4 + HS * 4 + 2 * ((nbmax + 7) & ~3) * 4 + 32 * 4 + HS * 2 + HS * 4 + HS * lt_bytes
    budget = min(device_attrs.smem_optin(), device_attrs._attr(_ATTR_SMEM_PER_SM, 0) // 2 - device_attrs._attr(_ATTR_SMEM_RESERVED, 0))
    cap = min((budget - tables) // lt_bytes, (1 << 18) - 16)
    if region > 0:
        cap = min(cap, region)
    cap = cap // 16 * 16
    assert cap >= 16
    return max(-(-m // cap) for m in seg_lens), nbmax


def _permute(g, n_cls, base, st, algo, region=0, lib=None, n_libs=0):
    plan = NhoodPlan(g.indptr, g.indices, n_cls)
    plan.set_option("shuffle_algo", algo)
    if algo >= 0:
        plan.set_option("shuffle_threads", NT if algo == 9 else 1024)
        plan.set_option("shuffle_r", 2)
    plan.set_option("shuffle_region", region)
    if lib is None:
        plan.set_base(base)
    else:
        plan.set_base(base, lib, n_libs)
    out = plan.permute(st)
    plan.upload(st)
    tail = plan.shuffled_labels(len(st) - 2, len(st))
    plan.close()
    return out, tail


def _check(g, n_cls, base, st, algo, region=0, lib=None, n_libs=0):
    got, tail = _permute(g, n_cls, base, st, algo, region, lib, n_libs)
    exp_tail = ref.shuffle_labels(base, st[-2:], lib, n_libs) if lib is not None else ref.shuffle_labels(base, st[-2:])
    np.testing.assert_array_equal(tail, exp_tail)
    exp, _ = _permute(g, n_cls, base, st, 7, region, lib, n_libs)
    np.testing.assert_array_equal(got, exp)


def _chain(n):
    return sp.csr_matrix((np.ones(n - 1, np.float32), (np.arange(n - 1), np.arange(1, n))), shape=(n, n))


def test_auto_more_step_blocks_than_threads_full_size():
    """1.21M spots (1100 x 1100 grid, 30 clusters) in auto mode: 591 step blocks for 512 threads, which the replay used to
    hand to the 1024-thread shape; more permutations than the grid's resident CTAs, so the persistent loop wraps."""
    g = synth.hex_graph(1100, 1100)
    n = g.shape[0]
    R, nbmax = _regions([n], 1)
    assert R <= RMAX and nbmax > NT, (R, nbmax)
    base = synth.categorical_labels(n, 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
    _check(g, 30, base, spawn_states(21, 2 * device_attrs.sm_count() + 8), -1)


@pytest.mark.parametrize("region", [31264, 48000])
def test_more_than_sixteen_regions_full_size(region):
    """configs[1] shape (1M spots) with 32 (the most a segment may take) and 21 regions of the given size."""
    g = synth.hex_graph(1000, 1000)
    n = g.shape[0]
    R, _ = _regions([n], 1, region)
    assert 16 < R <= RMAX, R
    base = synth.categorical_labels(n, 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
    _check(g, 30, base, spawn_states(22 + region, 12), 9, region)


def test_u16_labels_segments_many_regions_and_blocks():
    """16-bit labels (300 categories) over three library segments of unequal length, 1.15M elements in all: the longest
    segment takes more than 16 regions and more step blocks than threads."""
    n = 1_150_000
    g = _chain(n)
    lib = np.zeros(n, np.int32)
    lib[1_100_000:] = 1
    lib[1_140_000:] = 2
    R, nbmax = _regions([1_100_000, 40_000, 10_000], 2)
    assert 16 < R <= RMAX and nbmax > NT, (R, nbmax)
    base = (np.arange(n) * 13 % 300).astype(np.uint32)
    _check(g, 300, base, spawn_states(23, 4), 9, 0, lib, 3)


def test_many_permutations_small_array_many_regions():
    """More permutations than resident CTAs on a 70 001-element array in 30 regions: every CTA replays several permutations."""
    n = 70_001
    g = _chain(n)
    R, _ = _regions([n], 1, 2336)
    assert 16 < R <= RMAX, R
    base = (np.arange(n) * 13 % 30).astype(np.uint32)
    _check(g, 30, base, spawn_states(24, 6 * device_attrs.sm_count() + 5), 9, 2336)
