"""``mask_graph`` (``src/squidpy/gr/_build.py:853-966``): keep or drop the entries of a spatial graph by a polygon, on the GPU.

Every stored entry ``(i, j)`` of the connectivities is the segment ``coords[i] -> coords[j]``; the predicate is shapely's
``LineString.within(polygon)``, decided with exact orientation signs (``csrc/mask_pred.h``, DESIGN.md §3.12) instead of one
GEOS call per edge.  The polygon is read through ``__geo_interface__``, so shapely geometries work unchanged and shapely is
never imported.
"""

from __future__ import annotations

import ctypes as C
import sys
from typing import Any

import numpy as np

from .._constants import Key
from .._device import DevArray, DevSparse, _torch_stream, array_device, device_graph, device_matrix, graph_args, graph_value_code
from .._lib import check, default_context, load, pointer_device
from .._validators import extract_adata_if_sdata
from ._utils import _save_data

__all__ = ["mask_graph", "mask_csr", "host_mask"]

COORD_MIN, COORD_MAX = 2.0**-120, 2.0**120
_HOST_CODES = {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.int32): 3, np.dtype(np.int64): 4, np.dtype(np.bool_): 5}


def _in_range(a: np.ndarray) -> bool:
    m = np.abs(a)
    return bool(np.all((m == 0) | ((m >= COORD_MIN) & (m <= COORD_MAX))))


def polygon_rings(polygon_mask: Any) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The rings of a ``Polygon`` / ``MultiPolygon`` (``__geo_interface__``) as ``(xy float64[m, 2], ptr int64[r + 1], hole uint8[r])``:
    x and y only, every polygon's shell first, then its holes."""
    gi = getattr(polygon_mask, "__geo_interface__", None)
    kind = gi.get("type") if isinstance(gi, dict) else None
    if kind not in ("Polygon", "MultiPolygon"):
        raise ValueError(f"`polygon_mask` should be of type `Polygon` or `MultiPolygon`, got {type(polygon_mask)}")
    polys = [gi["coordinates"]] if kind == "Polygon" else list(gi["coordinates"])
    xy, ptr, hole = [], [0], []
    for poly in polys:
        for k, ring in enumerate(poly):
            a = np.asarray([tuple(v)[:2] for v in ring], dtype=np.float64).reshape(-1, 2)
            xy.append(a)
            ptr.append(ptr[-1] + a.shape[0])
            hole.append(int(k > 0))
    xy_arr = np.ascontiguousarray(np.concatenate(xy) if xy else np.empty((0, 2)), dtype=np.float64)
    if not (np.isfinite(xy_arr).all() and _in_range(xy_arr)):
        raise ValueError("Polygon vertices must be finite and 0 or of magnitude in [2^-120, 2^120].")
    return xy_arr, np.asarray(ptr, dtype=np.int64), np.asarray(hole, dtype=np.uint8)


def _check_host_graph(m: Any, n: int, what: str) -> None:
    """A host graph must be an ``n x n`` scipy CSR of a supported value dtype storing every ``(row, col)`` at most once."""
    import scipy.sparse as sp

    if not sp.issparse(m) or m.format != "csr":
        fmt = m.format if sp.issparse(m) else type(m).__name__
        raise ValueError(f"`mask_graph` reads the {what} as a CSR matrix, found `{fmt}`; convert it with `.tocsr()`.")
    if m.shape != (n, n):
        raise ValueError(f"Expected the {what} to be of shape `{(n, n)}`, found `{m.shape}`.")
    if np.dtype(m.dtype) not in _HOST_CODES:
        raise TypeError(f"Graph values of dtype `{m.dtype}` are not supported; use float32, float64, int32, int64 or bool.")
    ip, ix = np.asarray(m.indptr, dtype=np.int64), np.asarray(m.indices, dtype=np.int64)
    # a row stored in ascending columns cannot repeat one; only the other rows are searched
    starts = np.zeros(ix.size, dtype=bool)
    starts[ip[:-1][ip[:-1] < ix.size]] = True
    if ix.size > 1 and not np.all((np.diff(ix) > 0) | starts[1:]):
        rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(ip))
        if np.unique(rows * n + ix).size != ix.size:
            raise ValueError(f"The {what} store a (row, col) entry more than once; call `sum_duplicates()` first.")


def _host_args(m: Any):
    """The graph arguments of ``sqb_mask_graph`` for a checked host CSR, and the arrays behind them."""
    ip, ix = (np.ascontiguousarray(a) if a.dtype in (np.int32, np.int64) else np.ascontiguousarray(a, np.int64) for a in (m.indptr, m.indices))
    data = np.ascontiguousarray(m.data)
    return (ix.size, ip.ctypes.data, 8 * ip.itemsize, ix.ctypes.data, 8 * ix.itemsize, data.ctypes.data, _HOST_CODES[np.dtype(m.dtype)]), (ip, ix, data)


def _device_graph(d: DevSparse, n: int, what: str):
    if d.format != "csr":
        raise ValueError(f"`mask_graph` reads the {what} as a CSR matrix, found a device `{d.format}`.")
    g = graph_args(d, n)
    code = graph_value_code(d.data, g.nnz)
    if code == 2:
        raise TypeError(f"Device graph values of dtype `float16` are not supported; use float32, float64, int32, int64 or bool.")
    return (g.nnz, g.indptr, g.indptr_bits, g.indices or None, g.index_bits, d.data.ptr or None, code), g.stream, d


def _coords(coords: Any, n: int):
    """``(xy arguments of sqb_mask_graph, owner, device or None)``."""
    d = device_matrix(coords)
    if d is None:
        xy = np.asarray(coords)
        if xy.ndim != 2 or xy.shape[1] != 2:
            raise NotImplementedError(f"`mask_graph` takes 2-D coordinates (n, 2), found shape `{xy.shape}`.")
        xy = np.ascontiguousarray(xy, dtype=np.float64)
        if xy.shape[0] != n:
            raise ValueError(f"Expected `{n}` coordinates, found `{xy.shape[0]}`.")
        bad = np.flatnonzero(~np.isfinite(xy).all(axis=1))
        if bad.size:
            raise ValueError(f"coordinates of observation {bad[0]} are not finite")
        if not _in_range(xy):
            raise ValueError("coordinates must be 0 or of magnitude in [2^-120, 2^120]")
        return (xy.ctypes.data, 1, 2, 1, 0, 0), xy, None
    if not isinstance(d, DevArray):
        raise NotImplementedError("Spatial coordinates must be a dense (n, 2) array, found a sparse device matrix.")
    if len(d.shape) != 2 or d.shape[1] != 2:
        raise NotImplementedError(f"`mask_graph` takes 2-D coordinates (n, 2), found shape `{d.shape}`.")
    if d.shape[0] != n:
        raise ValueError(f"Expected `{n}` coordinates, found `{d.shape[0]}`.")
    if d.dtype not in (np.dtype(np.float32), np.dtype(np.float64)):
        raise TypeError(f"Device coordinates of dtype `{d.dtype}` are not supported; use float32 or float64.")
    return (d.ptr, int(d.dtype == np.float64), d.strides[0], d.strides[1], 1, d.stream), d, array_device(d, pointer_device)


def mask_csr(adj: Any, dst: Any, coords: Any, rings: tuple[np.ndarray, np.ndarray, np.ndarray], negative: bool, *,
             device: int | None = None) -> tuple[Any, Any]:
    """The masked ``(adj, dst)`` on the GPU (``sqb_mask_graph``): scipy CSRs with the inputs' index dtypes for host graphs, torch
    ``sparse_csr`` tensors on the graphs' device for device graphs.  ``rings``: ``polygon_rings`` of the polygon."""
    n = int(adj.shape[0])
    xy = _coords(coords, n)
    da, dd = device_graph(adj), device_graph(dst)
    if (da is None) != (dd is None):
        raise ValueError("The connectivities and the distances must both be on the host or both in GPU memory.")
    if da is None:
        _check_host_graph(adj, n, "connectivities")
        _check_host_graph(dst, n, "distances")
        if xy[2] is None:
            return host_mask(adj, dst, xy[1], rings, negative, device=device)
    return _mask(adj, dst, xy, rings, negative, device)


def host_mask(adj: Any, dst: Any, xy: np.ndarray, rings: tuple[np.ndarray, np.ndarray, np.ndarray], negative: bool, *,
              device: int | None = None) -> tuple[Any, Any]:
    """``mask_csr`` of checked host inputs: scipy CSRs ``adj`` / ``dst`` and C-contiguous float64 ``(n, 2)`` coordinates ``xy``."""
    return _mask(adj, dst, ((xy.ctypes.data, 1, 2, 1, 0, 0), xy, None), rings, negative, device)


def _mask(adj: Any, dst: Any, xy: tuple, rings: tuple[np.ndarray, np.ndarray, np.ndarray], negative: bool, device: int | None):
    """``sqb_mask_graph`` on checked inputs; ``xy``: what ``_coords`` returns."""
    n = int(adj.shape[0])
    xy_args, xy_keep, xy_dev = xy
    da, dd = device_graph(adj), device_graph(dst)
    on = None
    if da is not None:
        a_args, a_stream, a_src = _device_graph(da, n, "connectivities")
        d_args, d_stream, d_src = _device_graph(dd, n, "distances")
        on = array_device(da, pointer_device)
        if array_device(dd, pointer_device) != on:
            raise ValueError("The connectivities and the distances live on different devices.")
        if a_stream and d_stream and a_stream != d_stream:
            raise ValueError("The connectivities and the distances name different producer streams.")
        g_stream = a_stream or d_stream
    else:
        (a_args, a_keep), (d_args, d_keep) = _host_args(adj), _host_args(dst)
        a_src, d_src = adj, dst
        g_stream = 0
    for where in (on, xy_dev):
        if where is not None and device is not None and int(device) != where:
            raise ValueError(f"`device={device}` does not match the device of the graph or the coordinates, cuda:{where}.")
    if on is not None and xy_dev is not None and on != xy_dev:
        raise ValueError(f"The graph (cuda:{on}) and the coordinates (cuda:{xy_dev}) live on different devices.")
    on = on if on is not None else xy_dev if xy_dev is not None else device
    rxy, rptr, rhole = rings
    ctx = default_context(on)
    lib = load()
    h, na, nd = C.c_void_p(), C.c_int64(), C.c_int64()
    with ctx.lock:
        check(lib.sqb_mask_graph(ctx.handle, n, *a_args, *d_args, int(da is not None), g_stream, *xy_args, rxy.ctypes.data, rptr.ctypes.data,
                                 rhole.ctypes.data, rhole.size, int(bool(negative)), C.byref(h), C.byref(na), C.byref(nd)))
        try:
            if da is None:
                out = [(np.empty(n + 1, np.int32), np.empty(k.value, np.int32), np.empty(k.value, src.dtype)) for k, src in ((na, a_src), (nd, d_src))]
                check(lib.sqb_mask_export(h, *(a.ctypes.data for a in out[0]), *(a.ctypes.data for a in out[1]), 0))
            else:
                torch = sys.modules["torch"]
                tdev = torch.device("cuda", on)
                dt = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64, np.dtype(np.int32): torch.int32,
                      np.dtype(np.int64): torch.int64, np.dtype(np.bool_): torch.bool}
                out = [(torch.empty(n + 1, dtype=torch.int32, device=tdev), torch.empty(k.value, dtype=torch.int32, device=tdev),
                        torch.empty(k.value, dtype=dt[src.data.dtype], device=tdev)) for k, src in ((na, a_src), (nd, d_src))]
                check(lib.sqb_mask_export(h, *(t.data_ptr() or None for t in out[0]), *(t.data_ptr() or None for t in out[1]),
                                          _torch_stream(out[0][0])))
        finally:
            lib.sqb_mask_free(h)
    del xy_keep
    if da is None:
        return tuple(_host_csr(parts, src, n) for parts, src in zip(out, (a_src, d_src)))
    res = []
    for (ip, ix, v), src in zip(out, (a_src, d_src)):
        if 64 in (8 * src.indptr.dtype.itemsize, 8 * src.indices.dtype.itemsize):
            ip, ix = ip.to(torch.int64), ix.to(torch.int64)
        res.append(torch.sparse_csr_tensor(ip, ix, v, size=(n, n)))
    return tuple(res)


def _host_csr(parts, src, n: int):
    """A scipy CSR of the exported arrays with the index dtype of the source ``src``."""
    from scipy.sparse import csr_matrix

    ip, ix, v = parts
    m = csr_matrix((v, ix, ip), shape=(n, n))
    m.indptr, m.indices = ip.astype(src.indptr.dtype, copy=False), ix.astype(src.indices.dtype, copy=False)
    return m


def mask_graph(sdata: Any, table_key: str, polygon_mask: Any, negative_mask: bool = False, spatial_key: str = Key.obsm.spatial,
               key_added: str = "mask", copy: bool = False, *, device: int | None = None) -> tuple[Any, Any] | None:
    """Mask the spatial graph with a polygon (``_build.py:853-966``).

    Every stored entry ``(i, j)`` of ``obsp['{spatial_key}_connectivities']`` is the segment from ``obsm[spatial_key][i]`` to
    ``obsm[spatial_key][j]``.  It is *within* ``polygon_mask`` when no point of it lies outside the polygon and some point of its
    open part lies inside (shapely's ``LineString.within``): a segment that only runs along the boundary is not within, one that
    starts on the boundary and enters the polygon is.  A zero-length segment (a diagonal entry, or two observations at the same
    place) is its point: within iff the point is inside the polygon, not on its boundary (the point rule of GEOS's RelateNG;
    older GEOS releases may decide such segments differently).  The decisions are exact: orientation signs evaluated with
    adaptive-precision arithmetic, no constructed intersection point.

    ``negative_mask=False`` keeps the entries within the polygon, ``True`` drops them.  The distances lose the entries at the
    same ``(row, col)`` positions, then both matrices lose every zero-valued entry as scipy's ``eliminate_zeros`` does (a zero
    distance between coincident observations goes even when its edge is kept).  Values, their dtype and the order of the
    columns in every row are unchanged.

    ``polygon_mask`` is any object whose ``__geo_interface__`` is a ``Polygon`` or ``MultiPolygon`` (shapely's are); only x and y
    are read.  It must be valid (shapely's ``is_valid``); an empty polygon contains no edge.  Coordinates and polygon vertices
    must be 0 or of magnitude in ``[2^-120, 2^120]``.

    Unlike the reference, the source graph ``obsp['{spatial_key}_connectivities']`` (``uns[...]['unfiltered_graph_key']``) and
    the distances are left unmodified.  Host graphs (scipy CSR) give scipy CSRs with the input's index dtype; graphs in GPU
    memory (torch ``sparse_csr`` or cupyx-style CSR) give torch ``sparse_csr`` tensors on that device, equal to the host result.
    CSC graphs and graphs storing a ``(row, col)`` twice raise ``ValueError``.

    Returns ``(adj, dst)`` if ``copy``; else writes ``obsp['{key_added}_{spatial_key}_connectivities']``,
    ``obsp['{key_added}_{spatial_key}_distances']`` and ``uns['{key_added}_{spatial_key}_neighbors']`` and returns ``None``.
    """
    neighs_key = Key.uns.spatial_neighs(spatial_key)
    conns_key = Key.obsp.spatial_conn(spatial_key)
    dists_key = Key.obsp.spatial_dist(spatial_key)
    rings = polygon_rings(polygon_mask)
    table = extract_adata_if_sdata(sdata, table_key=table_key)
    adj, dst = mask_csr(table.obsp[conns_key], table.obsp[dists_key], table.obsm[spatial_key], rings, negative_mask, device=device)
    mask_conns_key = f"{key_added}_{conns_key}"
    mask_dists_key = f"{key_added}_{dists_key}"
    mask_neighs_key = f"{key_added}_{neighs_key}"
    neighbors_dict = {
        "connectivities_key": mask_conns_key,
        "distances_key": mask_dists_key,
        "unfiltered_graph_key": conns_key,
        "params": {"negative_mask": negative_mask, "table_key": table_key},
    }
    if copy:
        return adj, dst
    _save_data(table, attr="obsp", key=mask_conns_key, data=adj)
    _save_data(table, attr="obsp", key=mask_dists_key, data=dst, prefix=False)
    _save_data(table, attr="uns", key=mask_neighs_key, data=neighbors_dict, prefix=False)
    return None
