"""CPU restatement of the partition warp of the partitioned target generation (squidpy_b200/csrc/nhood.cu, 2f PART,
nhood_part_warp): the division-free region of a target, and the lane-parallel stable partition of a 2048-step block, checked
against the layout tests/emu_partition.py specifies."""
from __future__ import annotations

import random

import numpy as np
import pytest

from tests.emu_partition import SHIFT, partition_targets

L = 2048
RMAX = 16


def part_magic(B):
    """sqb_part_magic: region = umulhi(j, M) >> sh."""
    sh = (B - 1).bit_length() - 1
    M = ((1 << (32 + sh)) + B - 1) // B
    assert M < (1 << 32)
    return M, sh


def test_region_magic_is_exact_for_every_region_size():
    """Every region size sqb_part_regions can return (multiples of 16 below 2^18) and every target a segment of at most 16
    such regions holds, and at least every j < 2^20.  umulhi(j, M) >> sh never falls below j // B and never decreases in j,
    so it is exact on [kB, (k+1)B) iff it is exact at (k+1)B - 1: those are the values checked."""
    for B in range(16, 1 << 18, 16):
        M, sh = part_magic(B)
        jmax = max(1 << 20, RMAX * B)
        j = np.arange(B - 1, jmax + B, B, dtype=np.uint64)
        got = ((j * np.uint64(M)) >> np.uint64(32)) >> np.uint64(sh)
        np.testing.assert_array_equal(got, j // np.uint64(B), err_msg=f"B={B}")


def lane_chunk_partition(J, m, B):
    """The partition warp's build of the layout: lane l owns the steps t in [64 l, 64 l + 64) of the block, counts them per
    region, takes its slots from the region bases plus the counts of the higher lanes (earlier steps), and scatters its
    entries in step order (descending t)."""
    M, sh = part_magic(B)
    R = (m - 1) // B + 1
    P = [0] * m
    counts = []
    for b in range((m + L - 1) // L):
        bL, t0, t1 = b * L, 1 if b == 0 else 0, min(L, m - b * L)
        own = [range(max(t0 - 64 * lane, 0), min(t1 - 64 * lane, 64)) for lane in range(32)]
        region = lambda t: (J[bL + t] * M >> 32) >> sh  # noqa: E731
        cnt = [[0] * RMAX for _ in range(32)]
        for lane in range(32):
            for s in own[lane]:
                cnt[lane][region(64 * lane + s)] += 1
        tot = [sum(cnt[lane][r] for lane in range(32)) for r in range(RMAX)]
        for lane in range(32):
            slot = [sum(tot[:r]) + sum(cnt[hl][r] for hl in range(lane + 1, 32)) for r in range(RMAX)]
            for s in reversed(own[lane]):
                t = 64 * lane + s
                r = region(t)
                P[bL + slot[r]] = (t << SHIFT) | (J[bL + t] - r * B)
                slot[r] += 1
        assert all(c == 0 for c in tot[R:])
        counts.append(tot[:R])
    return P, counts


@pytest.mark.parametrize("m", [2, 3, 65, 2047, 2048, 2049, 6001])
def test_lane_chunk_partition_equals_specified_layout(m):
    rnd = random.Random(m)
    J = [0] + [rnd.randint(0, i) for i in range(1, m)]
    for R in (1, 2, 7, 16):
        B = ((m + R - 1) // R + 15) // 16 * 16  # sqb_part_regions with a cap that gives R regions
        assert lane_chunk_partition(J, m, B) == partition_targets(J, m, B, L)
