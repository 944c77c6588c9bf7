"""numpy restatement of ``sqb_window_ranges`` (``csrc/windows.cu``), test infrastructure: per window of each library and axis,
the comparisons ``end < v`` and ``start <= v`` the binary searches count, one window at a time as in the reference's loop."""

from __future__ import annotations

import numpy as np


def window_ranges(xy: np.ndarray, lib: np.ndarray, edge_off: np.ndarray, starts: np.ndarray, ends: np.ndarray) -> np.ndarray:
    """int32 (n, 4) ``[lo_x, hi_x, lo_y, hi_y]``: ``lo`` = number of windows whose end < v, ``hi`` = number whose start <= v,
    minus one; ``[0, -1, 0, -1]`` for ``lib = -1``."""
    xy = np.asarray(xy).reshape(-1, 2)
    lib = np.asarray(lib)
    out = np.tile(np.array([0, -1, 0, -1], dtype=np.int32), (xy.shape[0], 1))
    for code in range(len(edge_off) // 2):
        rows = np.flatnonzero(lib == code)
        for axis in (0, 1):
            v = xy[rows, axis]
            lo = np.zeros(rows.size, dtype=np.int32)
            hi = np.full(rows.size, -1, dtype=np.int32)
            for j in range(edge_off[2 * code + axis], edge_off[2 * code + axis + 1]):
                lo += ends[j] < v
                hi += starts[j] <= v
            out[rows, 2 * axis] = lo
            out[rows, 2 * axis + 1] = hi
    return out


def membership(ranges: np.ndarray, nx: int, ny: int) -> np.ndarray:
    """bool (n, nx * ny): observation i in window ix * ny + iy of its library, from its ranges."""
    lo_x, hi_x, lo_y, hi_y = (ranges[:, k, None] for k in range(4))
    ix, iy = np.divmod(np.arange(nx * ny), ny) if ny else (np.zeros(0, int), np.zeros(0, int))
    return (lo_x <= ix) & (ix <= hi_x) & (lo_y <= iy) & (iy <= hi_y)
