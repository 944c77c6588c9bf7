"""CPU restatement, word for word, of the two scans that let a segment take up to 32 regions (squidpy_b200/csrc/nhood.cu):
the partition warp's slot scan (2f PART, nhood_part_warp: per-lane u16 region counts packed two regions a 32-bit word, 16
words, or 8 when no segment has more than 16 regions, a suffix scan over the lanes by shuffles) and the region replay's run prefix (2j, nhood_apply_part_kernel: more step
blocks than threads, each thread taking ceil(nblk / NT) consecutive blocks).  Both are checked against the layout
tests/emu_partition.py specifies."""
from __future__ import annotations

import random

import numpy as np
import pytest

from tests.emu_partition import SHIFT, partition_targets

L = 2048
RMAX = 32
MASK32 = 0xFFFFFFFF


def part_magic(B):
    sh = (B - 1).bit_length() - 1
    return ((1 << (32 + sh)) + B - 1) // B, sh


def test_region_magic_is_exact_for_thirty_two_regions():
    """The division-free region stays exact over 32 regions of every region size (multiples of 16 below 2^18)."""
    for B in range(16, 1 << 18, 16):
        M, sh = part_magic(B)
        assert M < (1 << 32)
        j = np.arange(B - 1, RMAX * B + B, B, dtype=np.uint64)  # the last value of every region (see test_part_magic.py)
        got = ((j * np.uint64(M)) >> np.uint64(32)) >> np.uint64(sh)
        np.testing.assert_array_equal(got, j // np.uint64(B), err_msg=f"B={B}")


def warp_partition(J, m, B):
    """nhood_part_warp on one segment: returns (P, count rows of RMAX u16 counts)."""
    M, sh = part_magic(B)
    RW = 8 if (m - 1) // B + 1 <= 16 else RMAX // 2  # packed words the scan takes
    P = [0] * m
    rows = []
    for b in range((m + L - 1) // L):
        bL, t0, t1 = b * L, 1 if b == 0 else 0, min(L, m - b * L)
        s_rng = [(max(t0 - 64 * lane, 0), min(t1 - 64 * lane, 64)) for lane in range(32)]
        region = lambda t: ((J[bL + t] * M) >> 32) >> sh  # noqa: E731
        tab = [[0] * 32 for _ in range(RMAX)]  # tab[r][lane], u16
        for lane in range(32):
            for s in range(*s_rng[lane]):
                tab[region(64 * lane + s)][lane] += 1
        for r in range(RMAX):
            assert all(c <= 64 for c in tab[r])
        # w[k] = regions 2k (low half) and 2k + 1 (high half) of the lane
        w = [[tab[2 * k][lane] | (tab[2 * k + 1][lane] << 16) if k < RW else 0 for k in range(RMAX // 2)] for lane in range(32)]
        x = [list(wl) for wl in w]
        d = 1
        while d < 32:  # __shfl_down_sync suffix scan over the lanes
            y = [list(xl) for xl in x]
            for lane in range(32):
                if lane + d < 32:
                    for k in range(RW):
                        x[lane][k] = (x[lane][k] + y[lane + d][k]) & MASK32
            d <<= 1
        tot = [x[0][k] if k < RW else 0 for k in range(RMAX // 2)]
        for lane in range(32):
            run = 0
            for k in range(RW):
                lo = tot[k] & 0xFFFF
                slot = ((run | ((run + lo) << 16)) + x[lane][k] - w[lane][k]) & MASK32
                run += lo + (tot[k] >> 16)
                tab[2 * k][lane] = slot & 0xFFFF
                tab[2 * k + 1][lane] = slot >> 16
                assert tab[2 * k][lane] <= L and tab[2 * k + 1][lane] <= L  # u16 slots
        rows.append([(tot[r >> 1] >> ((r & 1) * 16)) & 0xFFFF for r in range(RMAX)])
        for lane in range(32):
            s0, s1 = s_rng[lane]
            for s in range(s1 - 1, s0 - 1, -1):
                t = 64 * lane + s
                r = region(t)
                slot = tab[r][lane]
                tab[r][lane] = (slot + 1) & 0xFFFF
                P[bL + slot] = (t << SHIFT) | (J[bL + t] - r * B)
    return P, rows


@pytest.mark.parametrize("m", [2, 65, 2049, 6001, 20000])
def test_warp_partition_32_regions_equals_specified_layout(m):
    rnd = random.Random(m)
    J = [0] + [rnd.randint(0, i) for i in range(1, m)]
    for R in (1, 15, 17, 26, 32):
        if R > m:
            continue
        B = ((m + R - 1) // R + 15) // 16 * 16  # sqb_part_regions with a cap that gives R regions
        R_eff = (m - 1) // B + 1
        P, rows = warp_partition(J, m, B)
        expP, expc = partition_targets(J, m, B, L)
        assert P == expP, (m, R)
        assert [row[:R_eff] for row in rows] == expc and all(c == 0 for row in rows for c in row[R_eff:])


def run_prefix_threads(rows, r, bt, nblk, NT):
    """The run scan of region r: block index t is block bt - t; thread tid takes [tid * per, tid * per + per).  Returns
    (s_bpref[0 .. nblk], s_bslot[0 .. nblk - 1])."""
    per = (nblk + NT - 1) // NT
    bpref, bslot = [None] * (nblk + 1), [None] * nblk
    sums, spans = [], []
    for tid in range(NT):
        t0, t1 = tid * per, min(tid * per + per, nblk)
        run = 0
        for t in range(t0, t1):
            b = bt - t
            pre, c_r = 0, 0
            for q in range((r >> 3) + 1):  # only the uint4 words region r's prefix needs
                for k in range(8):
                    c = rows[b][8 * q + k]
                    if 8 * q + k < r:
                        pre += c
                    if 8 * q + k == r:
                        c_r = c
            bpref[t], bslot[t] = run, b * L + pre
            run += c_r
        sums.append(run)
        spans.append((t0, t1))
    ex = 0
    for tid, (t0, t1) in enumerate(spans):  # the block-wide exclusive scan of the threads' sums
        for t in range(t0, t1):
            bpref[t] += ex
        if t0 < t1 and t1 == nblk:
            bpref[nblk] = ex + sums[tid]
        ex += sums[tid]
    return bpref, bslot


@pytest.mark.parametrize("NT,nblk", [(512, 1), (512, 489), (512, 512), (512, 513), (512, 591), (512, 1250), (1024, 1025), (8, 61)])
def test_run_prefix_with_more_blocks_than_threads(NT, nblk):
    rnd = random.Random(NT * 7919 + nblk)
    rows = [[rnd.choice([0, 0, rnd.randrange(0, 200)]) for _ in range(RMAX)] for _ in range(nblk)]
    bt = nblk - 1
    for r in (0, 7, 8, 16, 25, 31):
        bpref, bslot = run_prefix_threads(rows, r, bt, nblk, NT)
        runs = [rows[bt - t][r] for t in range(nblk)]
        assert bpref == [sum(runs[:t]) for t in range(nblk + 1)]
        assert bslot == [(bt - t) * L + sum(rows[bt - t][:r]) for t in range(nblk)]
