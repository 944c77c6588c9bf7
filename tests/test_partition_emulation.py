"""shuffle_algo 9 on the CPU (tests/emu_partition.py): the partitioned target layout round-trips, is what the streamed
per-block flush of nhood_jgen_kernel<Q, true> produces, and the region replay over it equals the plain Fisher-Yates sweep."""

from __future__ import annotations

import random

import pytest

from oracle import ref
from tests.emu_partition import partition_stream, partition_targets, region_replay_partitioned, unpack_targets
from tests.emu_shuffle import emu_targets, serial_targets


def _fisher_yates(arr, J):
    a = list(arr)
    for i in range(len(a) - 1, 0, -1):
        a[i], a[J[i]] = a[J[i]], a[i]
    return a


def _targets(rnd, m, mode):
    J = [0] * m
    for i in range(1, m):
        if mode == 0:  # uniform, like the real stream
            J[i] = rnd.randrange(i + 1)
        elif mode == 1:  # few distinct targets: long duplicate lists
            J[i] = min(i, rnd.choice([0, 1, 2, m // 3, m // 2]))
        elif mode == 2:  # targets close to the top: own-position chains
            J[i] = max(0, i - rnd.randrange(0, 4))
        else:  # everything aims at the lowest positions
            J[i] = rnd.randrange(min(i + 1, 6))
    return J


def test_partitioned_region_replay_equals_fisher_yates():
    """Any region size, block length and window length (tiny blocks and windows straddle block and region edges), uniform
    and adversarial targets."""
    rnd = random.Random(3)
    for trial in range(1500):
        m = rnd.choice([2, 3, 5, 17, 40, 97, 200, 333])
        J = _targets(rnd, m, trial % 4)
        arr = [rnd.randrange(1000) for _ in range(m)]
        B = rnd.choice([16, 32, 48, 64, 128, 1024])
        L = rnd.choice([4, 16, 32, 2048])
        P, counts = partition_targets(J, m, B, L)
        got = region_replay_partitioned(arr, P, counts, B, L, HS=rnd.choice([2, 8, 16, 64]), rng=rnd)
        assert got == _fisher_yates(arr, J), (trial, m, B, L)


def test_partition_round_trip_and_layout():
    rnd = random.Random(4)
    for trial in range(400):
        m = rnd.choice([2, 3, 33, 100, 1000, 5000])
        J = _targets(rnd, m, trial % 4)
        B = rnd.choice([16, 48, 256, 4096])
        L = rnd.choice([8, 64, 2048])
        P, counts = partition_targets(J, m, B, L)
        assert unpack_targets(P, counts, m, B, L) == J
        for b, row in enumerate(counts):  # every block holds exactly its own steps
            assert sum(row) == min(m, (b + 1) * L) - max(b * L, 1)
        assert all(e < (1 << 29) for e in P)  # 11-bit step offset (L <= 2048) + 18-bit region offset


@pytest.mark.parametrize("n", [2, 9, 2047, 2049, 5000, 20011])
def test_streamed_partition_of_generated_targets(n):
    """nhood_jgen_kernel's window sequence (emu_targets, generation order) flushed block by block equals the partition of
    numpy's target list; the replay over it gives numpy's shuffle."""
    st = ref.spawn_states(700 + n, 1)[0]
    state, inc = (int(st[0]) << 64) | int(st[1]), (int(st[2]) << 64) | int(st[3])
    gen = emu_targets(state, inc, [(0, n)], Q=4)
    J = [0] * n
    for (_, i), j in serial_targets(state, inc, [(0, n)]).items():
        J[i] = j
    for B, L in ((16 * ((n + 15) // 16), 2048), (48, 64), (1024, 2048)):
        if (n - 1) // B + 1 > 64:
            continue
        P, counts = partition_stream(((i, j) for (_, i), j in gen.items()), n, B, L)
        assert (P, counts) == partition_targets(J, n, B, L)
        arr = list(range(n))
        assert region_replay_partitioned(arr, P, counts, B, L, HS=32) == _fisher_yates(arr, J)
