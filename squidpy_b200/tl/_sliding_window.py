"""``sliding_window`` — drop-in for ``squidpy.tl.sliding_window`` (``src/squidpy/tl/_sliding_window.py:18-176``).

The reference builds one boolean mask over a library's observations per window and writes every window's observations into
the result by obs name (:130-158), a cost that grows as windows x observations.  Here the window edges are computed on the
host with the reference's numpy calls (:224-242; the device never recomputes an edge, so float32 minima, ``arange``'s
``start + i * step`` and the clipping are numpy's own values), and ONE call of ``sqb_window_ranges`` finds, for every
observation, the contiguous range of x windows and of y windows containing it, in the dtype numpy compares in.  The frame is
then built by position: the ordered categorical of the last window in index order (``overlap == 0``), or one object column of
``True`` / ``False`` per window (``overlap > 0``).

Obs names are assumed unique: with duplicates the reference's label-based ``.loc`` writes every row of a name, this does not.
"""

from __future__ import annotations

import time
from itertools import product
from typing import Any

import numpy as np
import pandas as pd

from .._device import on_host
from .._lib import Context, check, default_context, load
from .._validators import extract_adata_if_sdata
from ..gr._utils import _save_data, logg

__all__ = ["sliding_window", "window_ranges"]


def window_ranges(xy: np.ndarray, lib: np.ndarray, edge_off: np.ndarray, starts: np.ndarray, ends: np.ndarray, *,
                  ctx: Context | None = None) -> np.ndarray:
    """The windows containing every observation, on the GPU: int32 (n, 4) ``[lo_x, hi_x, lo_y, hi_y]``.

    ``xy`` is (n, 2) float64, or int64 when every edge and coordinate is an integer; ``lib`` int32 (n,) holds each
    observation's library in ``[-1, n_libs)`` (-1: none).  Library ``l``'s x edges are ``starts[edge_off[2l]:edge_off[2l+1]]``
    / ``ends[...]`` (same dtype as ``xy``, non-decreasing), its y edges the next range.  Observation ``i`` lies in window
    ``(ix, iy)`` of its library iff ``lo_x <= ix <= hi_x`` and ``lo_y <= iy <= hi_y``: an empty range on either axis, a NaN
    coordinate or ``lib = -1`` puts it in no window."""
    lib_ = load()
    ctx = ctx or default_context()
    dt = np.int64 if np.asarray(xy).dtype == np.int64 else np.float64
    xy_ = np.ascontiguousarray(np.asarray(xy, dtype=dt).reshape(-1, 2))
    lb = np.ascontiguousarray(np.asarray(lib, dtype=np.int32).reshape(-1))
    off = np.ascontiguousarray(np.asarray(edge_off, dtype=np.int64).reshape(-1))
    st = np.ascontiguousarray(np.asarray(starts, dtype=dt).reshape(-1))
    en = np.ascontiguousarray(np.asarray(ends, dtype=dt).reshape(-1))
    if lb.size != xy_.shape[0] or off.size % 2 != 1 or st.size != en.size or st.size != off[-1]:
        raise ValueError(f"window_ranges: {xy_.shape[0]} coordinates, {lb.size} library codes, {off.size} edge offsets ending at "
                         f"{off[-1] if off.size else None}, {st.size} starts and {en.size} ends do not fit together")
    out = np.empty((xy_.shape[0], 4), dtype=np.int32)
    check(lib_.sqb_window_ranges(ctx.handle, xy_.ctypes.data, int(dt is np.int64), xy_.shape[0], lb.ctypes.data, off.size // 2,
                                 off.ctypes.data, st.ctypes.data, en.ctypes.data, out.ctypes.data))
    return out


def _axis(lo: Any, hi: Any, window_size: int, overlap: int, drop_partial_windows: bool) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Every window start of one axis of ``_calculate_window_corners``, its end and whether it is kept: numpy's values and
    dtypes.  Ends are clipped to ``hi``, or left as they are when ``drop_partial_windows`` drops the windows beyond it."""
    starts = np.arange(lo, hi, window_size - overlap)
    ends = pd.Series(starts) + window_size
    if drop_partial_windows:
        return starts, ends.to_numpy(), (ends <= hi).to_numpy()
    return starts, ends.clip(upper=hi).to_numpy(), np.ones(starts.size, dtype=bool)


def _axis_windows(lo: Any, hi: Any, window_size: int, overlap: int, drop_partial_windows: bool) -> tuple[np.ndarray, np.ndarray]:
    """The starts and ends of the windows one axis keeps, in window order."""
    starts, ends, keep = _axis(lo, hi, window_size, overlap, drop_partial_windows)
    return starts[keep], ends[keep]


def _calculate_window_corners(min_x: int, max_x: int, min_y: int, max_y: int, window_size: int, overlap: int = 0,
                              drop_partial_windows: bool = False) -> pd.DataFrame:
    """The corners of every window covering ``[min_x, max_x] x [min_y, max_y]``: a frame with the columns ``x_start``,
    ``x_end``, ``y_start``, ``y_end``, one row per window, ``x`` windows outer and ``y`` windows inner.

    Windows start every ``window_size - overlap`` from the minimum up to (excluding) the maximum.  Border windows end at the
    maximum, or are dropped with ``drop_partial_windows``.  Raises ``ValueError`` for a negative ``overlap`` or one not
    smaller than ``window_size``."""
    if overlap < 0:
        raise ValueError("Overlap must be non-negative.")
    if overlap >= window_size:
        raise ValueError("Overlap must be less than the window size.")
    xs, xe, kx = _axis(min_x, max_x, window_size, overlap, drop_partial_windows)
    ys, ye, ky = _axis(min_y, max_y, window_size, overlap, drop_partial_windows)
    # the column dtypes are inferred from the rows of every window, before any is dropped
    windows = pd.DataFrame(list(product(xs, ys)), columns=["x_start", "y_start"])
    if len(windows):
        windows["x_end"], windows["y_end"] = np.repeat(xe, ys.size), np.tile(ye, xs.size)
        windows = windows[np.repeat(kx, ys.size) & np.tile(ky, xs.size)].reset_index(drop=True)
    else:
        windows["x_end"], windows["y_end"] = windows["x_start"] + window_size, windows["y_start"] + window_size
    return windows[["x_start", "x_end", "y_start", "y_end"]]


def _comparison_dtype(coord: np.dtype, edge: np.dtype) -> type:
    """The kernel dtype that orders a coordinate against an edge exactly as numpy's mixed-dtype comparison does."""
    ct = np.result_type(coord, edge)
    if ct.kind == "f" and ct.itemsize <= 8:
        return np.float64
    if ct.kind in "bi" or (ct.kind == "u" and ct.itemsize < 8):
        return np.int64
    raise NotImplementedError(f"sliding_window on the GPU compares float or integer coordinates, found {coord} against {edge} edges")


def sliding_window(
    adata: Any,
    library_key: str | None = None,
    window_size: int | None = None,
    overlap: int = 0,
    coord_columns: tuple[str, str] = ("globalX", "globalY"),
    sliding_window_key: str = "sliding_window_assignment",
    spatial_key: str = "spatial",
    drop_partial_windows: bool = False,
    copy: bool = False,
    *,
    table_key: str | None = None,
    device: int | None = None,
) -> pd.DataFrame | None:
    """Divide a tissue into square windows and assign every observation to them.

    Parameters as ``squidpy.tl.sliding_window``: coordinates come from ``adata.obs[list(coord_columns)]`` when both columns
    exist, else from the first two columns of ``adata.obsm[spatial_key]`` (host or device memory); windows of
    ``window_size`` (default ``max(floor(range // 3.95), 1)`` over all observations) start every ``window_size - overlap``
    from each library's minimum, per ``adata.obs[library_key]`` in order of first appearance.  A window holds the
    observations with ``start <= coordinate <= end`` on both axes; a NaN coordinate is in no window.  ``device``: the CUDA
    device (default: the context of ``squidpy_b200.default_context``).

    With ``overlap == 0`` the column ``sliding_window_key`` holds, per observation, the last window containing it as the ordered
    categorical ``"{library}_window_{i}"`` (``"window_{i}"`` without libraries); an observation in no window raises the
    reference's ``AttributeError``.  With ``overlap > 0`` every window is a column ``"{sliding_window_key}_{library}_window_{i}"``
    of ``True`` / ``False`` (object dtype).  The coordinate columns are appended.

    Returns the frame if ``copy=True``, else writes its columns into ``adata.obs``."""
    start = time.perf_counter()
    if overlap < 0:
        raise ValueError("Overlap must be non-negative.")
    adata = extract_adata_if_sdata(adata, table_key=table_key)
    obs = adata.obs

    x_col, y_col = coord_columns
    if x_col in obs and y_col in obs:
        coords = obs[[x_col, y_col]].copy()
    elif spatial_key in adata.obsm:
        coords = pd.DataFrame(np.asarray(on_host(adata.obsm[spatial_key]))[:, :2], index=obs.index, columns=[x_col, y_col])
    else:
        raise ValueError(f"Coordinates not found. Provide `{coord_columns}` in `adata.obs` or specify a suitable `spatial_key` in "
                         "`adata.obsm`.")
    cx, cy = coords[x_col], coords[y_col]

    if window_size is None:
        coord_range = max(cx.max() - cx.min(), cy.max() - cy.min())
        window_size = max(int(np.floor(coord_range // 3.95)), 1)
    if window_size <= 0:
        raise ValueError("Window size must be larger than 0.")
    if library_key is not None and library_key not in obs:
        raise ValueError(f"Library key '{library_key}' not found in adata.obs")
    libraries = [None] if library_key is None else obs[library_key].unique()
    if sliding_window_key in obs:
        logg.warning("Overwriting existing column '%s' in adata.obs.", sliding_window_key)

    # edges per library, on the host, with the reference's numpy calls
    n = len(obs)
    lib_code = np.zeros(n, dtype=np.int32) if library_key is None else np.full(n, -1, dtype=np.int32)
    axes: list[tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]] = []
    prefixes: list[str] = []
    vx, vy = cx.to_numpy(), cy.to_numpy()
    for code, lib in enumerate(libraries):
        if lib is not None:
            mask = np.asarray(obs[library_key] == lib, dtype=bool)
            lib_code[mask] = code
            lx, ly = pd.Series(vx[mask], copy=False), pd.Series(vy[mask], copy=False)  # pandas' min / max, without the obs index
        else:
            lx, ly = cx, cy
        if overlap >= window_size:
            raise ValueError("Overlap must be less than the window size.")
        axes.append(_axis_windows(lx.min(), lx.max(), window_size, overlap, drop_partial_windows)
                    + _axis_windows(ly.min(), ly.max(), window_size, overlap, drop_partial_windows))
        prefixes.append(f"{lib}_" if lib is not None else "")

    # the dtype the reference compares in: a window row (iterrows) takes the common dtype of its four edges, the coordinate
    # column is compared with that scalar
    edge_dt = np.result_type(*[a.dtype for ax in axes for a in ax if a.size]) if any(ax[0].size and ax[2].size for ax in axes) else np.float64
    kdt = _comparison_dtype(cx.dtype, edge_dt)
    if _comparison_dtype(cy.dtype, edge_dt) is not kdt:
        raise NotImplementedError(f"sliding_window on the GPU compares both axes in one dtype, found {cx.dtype} and {cy.dtype}")
    xy = np.empty((n, 2), dtype=kdt)
    xy[:, 0] = vx.astype(np.result_type(cx.dtype, edge_dt))
    xy[:, 1] = vy.astype(np.result_type(cy.dtype, edge_dt))
    edge_off, starts, ends = [0], [], []
    for xs, xe, ys, ye in axes:
        if xs.size == 0 or ys.size == 0:  # no windows in this library: no comparison is ever made
            xs = xe = ys = ye = np.zeros(0, dtype=kdt)
        for s, e in ((xs, xe), (ys, ye)):
            starts.append(s.astype(edge_dt).astype(kdt))
            ends.append(e.astype(edge_dt).astype(kdt))
            edge_off.append(edge_off[-1] + s.size)
    rng = window_ranges(xy, lib_code, np.asarray(edge_off), np.concatenate(starts) if starts else np.zeros(0, kdt),
                        np.concatenate(ends) if ends else np.zeros(0, kdt), ctx=default_context(device))
    lo_x, hi_x, lo_y, hi_y = rng.T

    cols: dict[str, Any] = {}
    if overlap == 0:
        # the last window in index order: (hi_x, hi_y); window ids are numbered over the libraries
        ny = np.array([ax[2].size for ax in axes], dtype=np.int64)
        first = np.concatenate([[0], np.cumsum([ax[0].size for ax in axes] * ny)]).astype(np.int64)
        if first[-1] == 0:  # the reference creates the column with its first window: without windows it has none to read
            raise KeyError(sliding_window_key)
        inside = (lo_x <= hi_x) & (lo_y <= hi_y)
        if not inside.all():  # an unassigned observation is NaN, which the reference's sort key cannot split
            raise AttributeError("'float' object has no attribute 'split'")
        wid = first[lib_code] + hi_x.astype(np.int64) * ny[lib_code] + hi_y
        seen = pd.unique(wid)  # order of first appearance in obs, stably sorted by the window's index in its library
        lib_of = np.searchsorted(first, seen, side="right") - 1
        local = seen - first[lib_of]
        order = np.argsort(local, kind="stable")
        pos = np.empty(first[-1], dtype=np.int64)
        pos[seen[order]] = np.arange(seen.size)
        labels = [f"{prefixes[lib_of[k]]}window_{local[k]}" for k in order]
        cols[sliding_window_key] = pd.Categorical.from_codes(pos[wid], categories=labels, ordered=True)
    else:
        for code, (xs, _, ys, _) in enumerate(axes):
            rows = np.flatnonzero(lib_code == code)
            lx, hx, ly, hy = lo_x[rows], hi_x[rows], lo_y[rows], hi_y[rows]
            for ix in range(xs.size):
                in_x = (lx <= ix) & (ix <= hx)
                for iy in range(ys.size):
                    col = np.zeros(n, dtype=bool)
                    col[rows] = in_x & (ly <= iy) & (iy <= hy)
                    cols[f"{sliding_window_key}_{prefixes[code]}window_{ix * ys.size + iy}"] = col.astype(object)
    df = pd.DataFrame(cols, index=obs.index)
    df[x_col] = coords[x_col]
    df[y_col] = coords[y_col]

    if copy:
        logg.info("Finish (%.3fs)", time.perf_counter() - start)
        return df
    for name, data in df.items():
        _save_data(adata, attr="obs", key=name, data=data)
    return None
