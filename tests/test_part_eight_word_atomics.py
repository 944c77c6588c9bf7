"""The partition warp's path for segments of at most 16 regions (squidpy_b200/csrc/nhood.cu 2f PART, nhood_part_warp<8>): a
32-bit region table per lane, counts and slots taken by shared-memory fetch-adds four steps at a time, and the stream-out of
the output block in 16-byte vectors when the block starts 16-byte aligned in J.  A CPU restatement of its loops, word for word,
against the layout tests/emu_partition.py specifies, and a GPU check of the shuffles it feeds at 14 and 16 regions, with
library segments that start on and off a 16-byte boundary."""
from __future__ import annotations

import random

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import NhoodPlan
from tests.emu_partition import SHIFT, partition_targets

L = 2048
MASK32 = 0xFFFFFFFF


def part_magic(B):
    sh = (B - 1).bit_length() - 1
    return ((1 << (32 + sh)) + B - 1) // B, sh


def warp_partition_8(J, m, B):
    """nhood_part_warp<8> on one segment: returns (P, count rows of 16 u16 counts)."""
    M, sh = part_magic(B)
    nB = -B & MASK32
    P = [None] * m
    rows = []
    for b in range((m + L - 1) // L):
        bL, t0, t1 = b * L, 1 if b == 0 else 0, min(L, m - b * L)
        tab = [[0] * 32 for _ in range(16)]  # tab32[r][lane]
        region = lambda t: ((J[bL + t] * M) >> 32) >> sh  # noqa: E731
        ranges = [(max(t0 - 64 * lane, 0), min(t1 - 64 * lane, 64)) for lane in range(32)]
        for lane, (s0, s1) in enumerate(ranges):  # count: batches of four, then the tail
            s = s0
            while s + 4 <= s1:
                for q in range(4):
                    tab[region(64 * lane + s + q)][lane] += 1
                s += 4
            while s < s1:
                tab[region(64 * lane + s)][lane] += 1
                s += 1
        w = [[tab[2 * k][lane] | (tab[2 * k + 1][lane] << 16) for k in range(8)] for lane in range(32)]
        x = [list(wl) for wl in w]
        d = 1
        while d < 32:
            y = [list(xl) for xl in x]
            for lane in range(32):
                if lane + d < 32:
                    for k in range(8):
                        x[lane][k] = (x[lane][k] + y[lane + d][k]) & MASK32
            d <<= 1
        tot = x[0]
        for lane in range(32):
            run = 0
            for k in range(8):
                lo = tot[k] & 0xFFFF
                slot = ((run | ((run + lo) << 16)) + x[lane][k] - w[lane][k]) & MASK32
                run += lo + (tot[k] >> 16)
                tab[2 * k][lane], tab[2 * k + 1][lane] = slot & 0xFFFF, slot >> 16
        rows.append([(tot[r >> 1] >> ((r & 1) * 16)) & 0xFFFF for r in range(16)])
        out = [None] * L
        for lane, (s0, s1) in enumerate(ranges):  # scatter in step order: batches of four, then the tail
            def put(slot, r, v):
                assert out[slot] is None
                out[slot] = (r * nB + v) & MASK32

            s = s1 - 1
            while s - 3 >= s0:
                rs = [region(64 * lane + s - q) for q in range(4)]
                slots = []
                for q in range(4):  # fetch-adds in step order
                    slots.append(tab[rs[q]][lane])
                    tab[rs[q]][lane] += 1
                ts = (64 * lane + s) << SHIFT
                for q in range(4):
                    put(slots[q], rs[q], J[bL + 64 * lane + s - q] + ts - (q << SHIFT))
                s -= 4
            while s >= s0:
                r = region(64 * lane + s)
                put(tab[r][lane], r, J[bL + 64 * lane + s] + ((64 * lane + s) << SHIFT))
                tab[r][lane] += 1
                s -= 1
        n = t1 - t0
        for aligned in (True, False):  # stream-out: every slot of the block exactly once, on either path
            written = []
            for lane in range(32):
                k = lane
                if aligned:
                    while k < n >> 2:
                        written += range(4 * k, 4 * k + 4)
                        k += 32
                    k = (n & ~3) + lane
                while k < n:
                    written.append(k)
                    k += 32
            assert sorted(written) == list(range(n))
        P[bL : bL + n] = out[:n]
    return [0 if p is None else p for p in P], rows


@pytest.mark.parametrize("m", [2, 3, 66, 130, 2049, 2050, 4163, 6001, 20000])
def test_eight_word_partition_equals_specified_layout(m):
    """Lanes own 0 to 64 steps (block 0 has no step 0, the last block is partial, and m - 1 is often no multiple of four)."""
    rnd = random.Random(m)
    J = [0] + [rnd.randint(0, i) for i in range(1, m)]
    for R in (1, 2, 13, 14, 15, 16):
        if R > m:
            continue
        B = ((m + R - 1) // R + 15) // 16 * 16  # sqb_part_regions with a cap that gives R regions
        R_eff = (m - 1) // B + 1
        assert R_eff <= 16
        P, rows = warp_partition_8(J, m, B)
        expP, expc = partition_targets(J, m, B, L)
        assert P == expP, (m, R)
        assert [row[:R_eff] for row in rows] == expc and all(c == 0 for row in rows for c in row[R_eff:])


def _chain(n):
    return sp.csr_matrix((np.ones(n - 1, np.float32), (np.arange(n - 1), np.arange(1, n))), shape=(n, n))


@pytest.mark.gpu
@pytest.mark.parametrize("region,R", [(3584, 14), (3136, 16)])
def test_eight_word_partition_shuffles_equal_numpy(region, R):
    """14 and 16 regions in the longest segment.  Library segments of 40 001, 50 003 and 29 997 labels start at 0, 40 001 and
    90 004 of the J row (rows start 16-byte aligned), so blocks take both stream-out paths.  The whole array as one segment
    is cut into 14 regions."""
    sizes = [40_001, 50_003, 29_997]
    n = sum(sizes)
    assert -(-max(sizes) // region) == R
    g = _chain(n)
    base = (np.arange(n) * 13 % 241).astype(np.uint32)
    lib = np.random.default_rng(R).permutation(np.repeat(np.arange(3, dtype=np.int32), sizes))
    for segs in (None, lib):
        plan = NhoodPlan(g.indptr, g.indices, 241)
        plan.set_option("shuffle_algo", 9)
        plan.set_option("shuffle_threads", 1024)
        plan.set_option("shuffle_region", region if segs is not None else 8592)  # 14 regions of the whole array
        if segs is None:
            plan.set_base(base)
        else:
            plan.set_base(base, segs, 3)
        st = spawn_states(R, 4)
        plan.upload(st)
        got = plan.shuffled_labels(0, 4)
        plan.close()
        exp = ref.shuffle_labels(base, st) if segs is None else ref.shuffle_labels(base, st, segs, 3)
        np.testing.assert_array_equal(got, exp)
