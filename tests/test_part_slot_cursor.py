"""The region replay's slot -> block lookup (squidpy_b200/csrc/nhood.cu 2j): each thread walks its block index forward from
the one it found one window back.  It must map every window slot to the block the binary search over the run prefix finds,
with empty runs anywhere and windows that start exactly on a block boundary."""

from __future__ import annotations

import random


def run_prefix(runs):
    """s_bpref of nhood_apply_part_kernel: exclusive prefix of one region's runs (runs[t] = the run of block bt - t, top block
    first), with the total at index len(runs)."""
    pref = [0]
    for c in runs:
        pref.append(pref[-1] + c)
    return pref


def slot_block_search(pref, g):
    """Block index t of window slot g < pref[-1] by binary search: the largest t < len(pref) - 1 with pref[t] <= g."""
    tl, th = 0, len(pref) - 1
    while th - tl > 1:
        mid = (tl + th) // 2
        if pref[mid] <= g:
            tl = mid
        else:
            th = mid
    return tl


def slot_blocks_cursor(pref, NT):
    """Block index of every slot as the kernel's threads find it: thread s owns the slots s + k NT + w HS (HS = 2 NT) of the
    windows w, for k = 0, 1, and walks its block index for slot k forward from the one it found for that slot one window
    back (from block 0 for the first window)."""
    total = pref[-1]
    HS = 2 * NT
    out = [None] * total
    for s in range(NT):
        for k in range(2):
            t = 0
            for g in range(s + k * NT, total, HS):
                while pref[t + 1] <= g:
                    t += 1
                out[g] = t
    return out


def _check(runs, NT):
    pref = run_prefix(runs)
    got = slot_blocks_cursor(pref, NT)
    assert got == [slot_block_search(pref, g) for g in range(pref[-1])], (runs, NT)
    for g, t in enumerate(got):  # the block's run holds the slot
        assert pref[t] <= g < pref[t + 1]


def test_cursor_equals_binary_search_random_runs():
    rnd = random.Random(7)
    for trial in range(300):
        NT = rnd.choice([1, 2, 4, 16, 64])
        nblk = rnd.randrange(1, 40)
        mode = trial % 3
        if mode == 0:  # sparse: most runs empty, including runs of empty blocks at either end
            runs = [rnd.choice([0, 0, 0, rnd.randrange(1, 50)]) for _ in range(nblk)]
        elif mode == 1:  # dense: runs much longer than a window
            runs = [rnd.randrange(0, 20 * NT + 1) for _ in range(nblk)]
        else:  # runs of whole windows, with empty blocks between: windows start exactly on block boundaries
            runs = [rnd.choice([0, 2 * NT, 4 * NT, NT]) for _ in range(nblk)]
        if sum(runs) == 0:
            runs[rnd.randrange(nblk)] = 1
        _check(runs, NT)


def test_cursor_equals_binary_search_kernel_shapes():
    """512 threads (1024-slot windows): runs shaped like one region's targets per 2048-step block, at 1M elements and 13
    regions, for the top and the bottom region, and with empty runs before and after."""
    rnd = random.Random(11)
    m, B, L = 1_000_000, 76_928, 2048
    for lo in (0, 12 * B):
        nblk = (m - 1) // L - lo // L + 1
        runs = [sum(1 for _ in range(L) if rnd.random() < min(1.0, B / max(m - t * L, 1))) for t in range(nblk)]
        _check(runs, 512)
        _check([0, 0] + runs + [0, 0, 0], 512)
