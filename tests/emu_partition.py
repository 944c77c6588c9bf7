"""Executable specification of shuffle_algo 9 (squidpy_b200/csrc/nhood.cu 2f PART and 2j): swap targets stored partitioned
by target region, one block of L consecutive steps at a time, and the region replay that consumes them.  Not used by the
product; tests/test_partition_emulation.py checks it against the plain Fisher-Yates sweep."""
from __future__ import annotations

import random

from tests.emu_shuffle import _resolve_general_window

SHIFT = 18  # entry = ((i - b*L) << SHIFT) | (j - region*B)


def _flush(block, b, L, B, R, P, counts):
    """block: the (i, j) pairs of block b in step order (descending i)."""
    groups = [[] for _ in range(R)]
    for i, j in block:
        r = j // B
        groups[r].append(((i - b * L) << SHIFT) | (j - r * B))
    k = b * L
    for r in range(R):
        counts[b][r] = len(groups[r])
        P[k : k + len(groups[r])] = groups[r]
        k += len(groups[r])


def partition_targets(J, m, B, L=2048):
    """Packed layout of the targets J[1..m-1] of one segment: block b keeps its entries in its own slots [bL, (b+1)L) of a
    J-sized list P, grouped by target region (region 0 first), in step order inside a region; counts[b][r] = entries of
    region r in block b.  Returns (P, counts)."""
    R = (m - 1) // B + 1
    nb = (m + L - 1) // L
    P = [0] * m
    counts = [[0] * R for _ in range(nb)]
    for b in range(nb):
        steps = range(min(m, (b + 1) * L) - 1, max(b * L, 1) - 1, -1)
        _flush([(i, J[i]) for i in steps], b, L, B, R, P, counts)
    return P, counts


def partition_stream(stream, m, B, L=2048):
    """The same layout built the way nhood_jgen_kernel<Q, true> builds it: (i, j) pairs arrive in generation order
    (descending i), are staged per block and flushed when the last step of the block has arrived."""
    R = (m - 1) // B + 1
    nb = (m + L - 1) // L
    P = [0] * m
    counts = [[0] * R for _ in range(nb)]
    blk, stage = (m - 1) // L, []
    for i, j in stream:
        assert i // L == blk
        stage.append((i, j))
        if i == max(blk * L, 1):
            _flush(stage, blk, L, B, R, P, counts)
            blk, stage = blk - 1, []
    assert not stage
    return P, counts


def unpack_targets(P, counts, m, B, L=2048):
    """Inverse of partition_targets: the plain target list J (J[0] = 0)."""
    J = [0] * m
    for b, row in enumerate(counts):
        k = b * L
        for r, c in enumerate(row):
            for e in P[k : k + c]:
                J[b * L + (e >> SHIFT)] = r * B + (e & ((1 << SHIFT) - 1))
            k += c
    return J


def region_replay_partitioned(arr, P, counts, B, L=2048, HS=16, rng=None):
    """Fisher-Yates steps i = m-1 .. 1 (swap i and J[i]) applied to a copy of `arr` one region [lo, hi) of B positions at a
    time, top region first, from the partitioned targets: region r's runs of the blocks from the top one down to the block of
    lo, concatenated in step order, in windows of exactly HS slots.  The slab of a region is read from the ORIGINAL labels:
    no pass writes a region before its own."""
    rng = rng or random.Random(0)
    a = list(arr)
    m = len(a)
    if m < 2:
        return a
    nb = len(counts)
    for r in range((m - 1) // B, -1, -1):
        lo = r * B
        hi = min(m, lo + B)
        assert a[lo:hi] == list(arr[lo:hi])
        slab = list(arr[lo:hi])
        tops, tgts = [], []
        for b in range(nb - 1, lo // L - 1, -1):
            k = b * L + sum(counts[b][:r])
            for e in P[k : k + counts[b][r]]:
                tops.append(b * L + (e >> SHIFT))
                tgts.append(lo + (e & ((1 << SHIFT) - 1)))
        for w0 in range(0, len(tops), HS):
            _resolve_general_window(slab, a, lo, hi, tops[w0 : w0 + HS], tgts[w0 : w0 + HS], rng)
        a[lo:hi] = slab
    return a
