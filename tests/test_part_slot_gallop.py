"""The region replay's slot -> block lookup as it now runs (squidpy_b200/csrc/nhood.cu 2j, block_of): each thread still walks
its block index forward from the one it found one window back, but four blocks a step, then two and one, over the run prefix
padded with the total.  It must find the same block as the binary search, with empty runs anywhere, windows starting on block
boundaries, and without reading past the three pad words."""

from __future__ import annotations

import random

from tests.test_part_slot_cursor import run_prefix, slot_block_search


def slot_blocks_gallop(pref, NT):
    total = pref[-1]
    nblk = len(pref) - 1
    padded = pref + [total] * 3  # s_bpref[nblk .. nblk + 3]
    HS = 2 * NT
    out = [None] * total

    def at(x):
        assert x <= nblk + 3, "read past the pad words"
        return padded[x]

    for s in range(NT):
        for k in range(2):
            t = 0
            for g in range(s + k * NT, total, HS):
                while at(t + 4) <= g:
                    t += 4
                if at(t + 2) <= g:
                    t += 2
                if at(t + 1) <= g:
                    t += 1
                out[g] = t
    return out


def _check(runs, NT):
    pref = run_prefix(runs)
    got = slot_blocks_gallop(pref, NT)
    assert got == [slot_block_search(pref, g) for g in range(pref[-1])], (runs, NT)


def test_gallop_equals_binary_search_random_runs():
    rnd = random.Random(13)
    for trial in range(400):
        NT = rnd.choice([1, 2, 4, 16, 64])
        nblk = rnd.randrange(1, 60)
        mode = trial % 3
        if mode == 0:
            runs = [rnd.choice([0, 0, 0, rnd.randrange(1, 50)]) for _ in range(nblk)]
        elif mode == 1:
            runs = [rnd.randrange(0, 20 * NT + 1) for _ in range(nblk)]
        else:
            runs = [rnd.choice([0, 2 * NT, 4 * NT, NT]) for _ in range(nblk)]
        if sum(runs) == 0:
            runs[rnd.randrange(nblk)] = 1
        _check(runs, NT)


def test_gallop_equals_binary_search_kernel_shape():
    """512 threads (1024-slot windows), 1M elements in 12 regions: the top and the bottom region's runs, and the same with
    empty runs before and after."""
    rnd = random.Random(17)
    m, B, L = 1_000_000, 83_344, 2048
    for lo in (0, 11 * B):
        nblk = (m - 1) // L - lo // L + 1
        runs = [sum(1 for _ in range(L) if rnd.random() < min(1.0, B / max(m - t * L, 1))) for t in range(nblk)]
        _check(runs, 512)
        _check([0, 0, 0, 0, 0] + runs + [0, 0, 0], 512)
