"""Spatial neighbour graphs on the GPU — drop-ins for ``squidpy.gr.spatial_neighbors_knn / _grid / _radius``
(``src/squidpy/gr/_build.py:484-549, 553-620, 701-786``) and the builder classes behind them
(``src/squidpy/gr/neighbors.py``: ``KNNBuilder`` :157-209, ``RadiusBuilder`` :212-270, ``GridBuilder`` :335-419), plus
``spatial_neighbors_delaunay`` / ``DelaunayBuilder`` (``_build.py:625-697``, ``neighbors.py:272-332``) and the public bridge
``spatial_neighbors_from_builder`` (``_build.py:388-460``).

This is the step right before every hot-path call (SURVEY.md 8f-1): at 1M spots the scikit-learn KD-tree query costs
seconds where the statistics now cost milliseconds.  The neighbour search runs on the H100 (``sqb_knn_2d`` /
``sqb_radius_2d``: exact, float64, scikit-learn's arithmetic, rows in CSR order); the cheap O(nnz) post-processing
(percentile / interval pruning, spectral / cosine transform, ring expansion, library block-diagonal) follows the
reference's scipy code on the host.  Output contract as in the reference: ``obsp['{key}_connectivities']`` CSR float32,
``obsp['{key}_distances']`` CSR, ``uns['{key}_neighbors']`` with the parameters.  The Delaunay graph is triangulated on the GPU
with exact predicates (``sqb_delaunay_2d``, DESIGN.md §3.10); ``GridBuilder(delaunay=True)`` still raises
``NotImplementedError``.

Coordinates already in GPU memory (a torch CUDA tensor or any ``__cuda_array_interface__`` exporter of shape (n, 2), float32
or float64, any strides) take the device path instead (``sqb_graph_build_device``): search AND post-processing run on the
GPU and both matrices are returned as torch ``sparse_csr`` CUDA tensors (int32 indices, ascending columns) that equal the
host path's result after ``sort_indices()`` bit for bit.  The coordinates are never read on the host.
"""

from __future__ import annotations

import ctypes as C
import time
from typing import Any, NamedTuple

import numpy as np
from scipy.sparse import block_diag, csr_matrix

from .._constants import CoordType, Key, Transform
from .._device import DevArray, _torch_stream, array_device, device_matrix
from .._lib import Context, check, default_context, load, pointer_device
from .._validators import assert_categorical_obs, assert_positive, assert_spatial_basis, extract_adata_if_sdata
from ._utils import _save_data, logg

__all__ = ["spatial_neighbors_knn", "spatial_neighbors_grid", "spatial_neighbors_radius", "spatial_neighbors_delaunay",
           "spatial_neighbors_from_builder", "SpatialNeighborsResult", "KNNBuilder", "GridBuilder", "RadiusBuilder", "DelaunayBuilder",
           "knn_2d", "radius_2d", "delaunay_2d"]


class SpatialNeighborsResult(NamedTuple):
    """Result of the ``spatial_neighbors_*`` functions (``_build.py:56-60``)."""

    connectivities: csr_matrix
    distances: csr_matrix


# ---------------------------------------------------------------------------------------------------------
# device searches
# ---------------------------------------------------------------------------------------------------------
def _coords2d(coords) -> np.ndarray:
    xy = np.ascontiguousarray(np.asarray(coords, dtype=np.float64))
    if xy.ndim != 2 or xy.shape[1] != 2:
        raise NotImplementedError(f"The GPU graph builders take 2-D coordinates (n, 2), found shape `{xy.shape}`.")
    return xy


def knn_2d(coords, k: int, *, median: bool = False, ctx: Context | None = None):
    """``NearestNeighbors(n_neighbors=k).fit(coords).kneighbors()`` on the GPU: ``(dist float64[n, k], idx int32[n, k])`` with
    every row ordered by ascending neighbour index (CSR order) — and ``np.median(dist)`` if ``median``."""
    xy = _coords2d(coords)
    n = xy.shape[0]
    ctx = ctx or default_context()
    idx = np.empty((n, k), dtype=np.int32)
    dist = np.empty((n, k), dtype=np.float64)
    med = C.c_double(0.0)
    with ctx.lock:
        check(load().sqb_knn_2d(ctx.handle, xy.ctypes.data, n, int(k), idx.ctypes.data, dist.ctypes.data, C.byref(med) if median else None))
    return (dist, idx, med.value) if median else (dist, idx)


def radius_2d(coords, radius: float, *, ctx: Context | None = None):
    """``NearestNeighbors(radius=r).fit(coords).radius_neighbors()`` on the GPU as CSR pieces: ``(indptr int64[n+1],
    idx int32[nnz], dist float64[nnz])``, rows in ascending column order."""
    xy = _coords2d(coords)
    n = xy.shape[0]
    ctx = ctx or default_context()
    lib = load()
    indptr = np.empty(n + 1, dtype=np.int64)
    nnz = C.c_int64(0)
    with ctx.lock:
        check(lib.sqb_radius_2d(ctx.handle, xy.ctypes.data, n, float(radius), indptr.ctypes.data, None, None, 0, C.byref(nnz)))
        idx = np.empty(max(nnz.value, 1), dtype=np.int32)
        dist = np.empty(max(nnz.value, 1), dtype=np.float64)
        check(lib.sqb_radius_2d(ctx.handle, xy.ctypes.data, n, float(radius), indptr.ctypes.data, idx.ctypes.data, dist.ctypes.data, idx.size, C.byref(nnz)))
    return indptr, idx[: nnz.value], dist[: nnz.value]


def delaunay_2d(coords, *, ctx: Context | None = None, pass_counts: bool = False):
    """``scipy.spatial.Delaunay(coords).vertex_neighbor_vertices`` on the GPU: ``(indptr int64[n+1], idx int32[nnz])`` with every
    row in ascending column order (and the points finished by pass 1 and pass 2 if ``pass_counts``).  Exact duplicates are
    collapsed to the lowest index of their group; the other copies get empty rows.  Raises ``scipy.spatial.QhullError`` for
    fewer than three distinct points or all of them collinear."""
    from scipy.spatial import QhullError

    xy = _coords2d(coords)
    if not np.isfinite(xy).all():
        raise ValueError("Points cannot contain NaN")
    n = xy.shape[0]
    if n >= 2**31 - 1:
        raise ValueError(f"Delaunay graphs take fewer than 2^31 - 1 points, found {n}.")
    ctx = ctx or default_context()
    indptr = np.empty(n + 1, dtype=np.int64)
    idx = np.empty(max(6 * n, 1), dtype=np.int32)  # a planar graph has fewer than 3n edges
    nnz, counts = C.c_int64(0), np.zeros(2, dtype=np.int64)
    with ctx.lock:
        try:
            check(load().sqb_delaunay_2d(ctx.handle, xy.ctypes.data, n, indptr.ctypes.data, idx.ctypes.data, idx.size, C.byref(nnz), counts.ctypes.data))
        except ValueError as e:
            if str(e).startswith("QhullError"):
                raise QhullError(str(e)) from None
            raise
    out = (indptr, idx[: nnz.value].copy())
    return (*out, counts) if pass_counts else out


def _device_coords(coords) -> DevArray | None:
    """The device description of coordinates in GPU memory, or ``None`` for host coordinates."""
    d = device_matrix(coords)
    if d is None:
        return None
    if not isinstance(d, DevArray):
        raise NotImplementedError("Spatial coordinates must be a dense (n, 2) array, found a sparse device matrix.")
    if len(d.shape) != 2 or d.shape[1] != 2:
        raise ValueError(f"Expected device coordinates of shape `(n, 2)`, found `{d.shape}`.")
    if d.dtype not in (np.dtype(np.float32), np.dtype(np.float64)):
        raise TypeError(f"Device coordinates of dtype `{d.dtype}` are not supported; use float32 or float64.")
    return d


_TRANSFORM_CODES = {Transform.NONE: 0, Transform.SPECTRAL: 1, Transform.COSINE: 2}


# ---------------------------------------------------------------------------------------------------------
# post-processing (host, O(nnz); follows neighbors.py:423-560)
# ---------------------------------------------------------------------------------------------------------
def _filter_by_radius_interval(adj: csr_matrix, dst: csr_matrix, radius: tuple[float, float]) -> None:
    minn, maxx = radius
    mask = (dst.data < minn) | (dst.data > maxx)
    a_diag = adj.diagonal()
    dst.data[mask] = 0.0
    adj.data[mask] = 0.0
    adj.setdiag(a_diag)


def _percentile(adj: csr_matrix, dst: csr_matrix, percentile: float) -> tuple[csr_matrix, csr_matrix]:
    threshold = np.percentile(dst.data, percentile)
    adj[dst > threshold] = 0.0
    dst[dst > threshold] = 0.0
    return adj, dst


def _transform_spectral(a: csr_matrix) -> csr_matrix:
    """D^-1/2 A D^-1/2 with D = column sums (``symmetric_normalize_csr``, neighbors.py:530-549), float32 result."""
    if not a.nnz:
        return a
    degrees = np.squeeze(np.array(np.sqrt(1.0 / a.sum(axis=0))))
    rows = np.repeat(np.arange(a.shape[0]), np.diff(a.indptr))
    res = (degrees[rows] * degrees[a.indices] * a.data).astype(np.float32)
    return csr_matrix((res, a.indices, a.indptr), shape=a.shape)


def _apply_transform(adj: csr_matrix, dst: csr_matrix, transform: Transform) -> tuple[csr_matrix, csr_matrix]:
    # eliminate_zeros() of the reference (neighbors.py:463-464); a full pass only when there is something to drop
    if np.count_nonzero(adj.data) != adj.data.size:
        adj.eliminate_zeros()
    if np.count_nonzero(dst.data) != dst.data.size:
        dst.eliminate_zeros()
    if transform == Transform.SPECTRAL:
        return _transform_spectral(adj), dst
    if transform == Transform.COSINE:
        from sklearn.metrics.pairwise import cosine_similarity

        return cosine_similarity(adj, dense_output=False), dst
    if transform == Transform.NONE:
        return adj, dst
    raise NotImplementedError(f"Transform `{transform}` is not yet implemented.")


# ---------------------------------------------------------------------------------------------------------
# builders (same constructor arguments / uns_params / build contract as neighbors.py)
# ---------------------------------------------------------------------------------------------------------
class _Builder:
    def __init__(self, transform=None, set_diag: bool = False, percentile: float | None = None, ctx: Context | None = None):
        self.transform = Transform.NONE if transform is None else Transform(transform)
        self.set_diag = set_diag
        self.percentile = percentile
        self.ctx = ctx

    def build_graph(self, coords) -> tuple[csr_matrix, csr_matrix]:  # pragma: no cover
        raise NotImplementedError

    def _interval(self):
        return None

    def _diagonals(self, adj: csr_matrix, dst: csr_matrix) -> None:
        """``adj.setdiag(1.0 if set_diag else adj.diagonal()); dst.setdiag(0.0)`` (neighbors.py:206-208, :267-269).  scipy stores
        the diagonal it is given EXPLICITLY (also zeros), and the percentile / interval post-processors look at ``.data`` before
        ``eliminate_zeros`` runs, so those cases replay the calls literally; otherwise the explicit zeros would only be
        inserted to be removed again (the searches never return the query itself) and are skipped."""
        if self.set_diag or self.percentile is not None or self._interval() is not None:
            adj.setdiag(1.0 if self.set_diag else adj.diagonal())
            dst.setdiag(0.0)

    def _device_args(self) -> tuple[int, int, int, float, tuple[float, float] | None]:  # pragma: no cover
        """(kind, n_neighbors, n_rings, radius, interval) of ``sqb_graph_build_device``."""
        raise NotImplementedError

    def build_device(self, d: DevArray, device: int | None = None, libraries: tuple[np.ndarray, np.ndarray] | None = None):
        """The graph of device coordinates ``d`` on their device (an explicit ``device`` must name it) as torch ``sparse_csr``
        CUDA tensors; ``libraries = (ptr int64, rows int32)`` builds every library's rows as its own block."""
        import torch

        on = array_device(d, pointer_device)
        if device is not None and int(device) != on:
            raise ValueError(f"`device={device}` does not match the device of the spatial coordinates, cuda:{on}.")
        ctx = self.ctx if self.ctx is not None and self.ctx.device == on else default_context(on)
        kind, k, n_rings, radius, interval = self._device_args()
        lo, hi = interval if interval is not None else (0.0, 0.0)
        pct = np.nan if self.percentile is None else float(self.percentile)
        lp, lr, n_libs = (None, None, 0) if libraries is None else (libraries[0].ctypes.data, libraries[1].ctypes.data, libraries[0].size - 1)
        lib = load()
        h, n_out, nnz_a, nnz_d, f64 = C.c_void_p(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int()
        with ctx.lock:
            check(lib.sqb_graph_build_device(ctx.handle, d.ptr, int(d.dtype == np.float64), d.shape[0], d.strides[0], d.strides[1], d.stream, kind, k,
                                             n_rings, float(radius), int(interval is not None), float(lo), float(hi), int(bool(self.set_diag)), pct,
                                             _TRANSFORM_CODES[self.transform], lp, lr, n_libs, C.byref(h), C.byref(n_out), C.byref(nnz_a),
                                             C.byref(nnz_d), C.byref(f64)))
            try:
                n, dev = n_out.value, torch.device("cuda", on)
                parts = [torch.empty(n + 1, dtype=torch.int32, device=dev), torch.empty(nnz_a.value, dtype=torch.int32, device=dev),
                         torch.empty(nnz_a.value, dtype=torch.float32, device=dev), torch.empty(n + 1, dtype=torch.int32, device=dev),
                         torch.empty(nnz_d.value, dtype=torch.int32, device=dev),
                         torch.empty(nnz_d.value, dtype=torch.float64 if f64.value else torch.float32, device=dev)]
                check(lib.sqb_graph_export(h, *(t.data_ptr() or None for t in parts), _torch_stream(parts[0])))
            finally:
                lib.sqb_graph_free(h)
        adj = torch.sparse_csr_tensor(parts[0], parts[1], parts[2], size=(n, n))
        dst = torch.sparse_csr_tensor(parts[3], parts[4], parts[5], size=(n, n))
        return adj, dst

    def build(self, coords) -> tuple[csr_matrix, csr_matrix]:
        d = _device_coords(coords)
        if d is not None:
            return self.build_device(d, None if self.ctx is None else self.ctx.device)
        return self._build_host(coords)

    def _build_host(self, coords) -> tuple[csr_matrix, csr_matrix]:
        import warnings

        from scipy.sparse import SparseEfficiencyWarning

        with warnings.catch_warnings():
            warnings.simplefilter("ignore", SparseEfficiencyWarning)
            adj, dst = self.build_graph(coords)
            if self._interval() is not None:
                _filter_by_radius_interval(adj, dst, self._interval())
            if self.percentile is not None:
                adj, dst = _percentile(adj, dst, self.percentile)
            return _apply_transform(adj, dst, self.transform)

    def combine(self, mats, ixs) -> tuple[csr_matrix, csr_matrix]:
        """Per-library blocks -> one graph in the original observation order (``GraphBuilderCSR.combine``, neighbors.py:138-156)."""
        adj = block_diag([m[0] for m in mats], format="csr")
        dst = block_diag([m[1] for m in mats], format="csr")
        ixs_arr = np.asarray(ixs)
        if ixs_arr.size and np.any(np.diff(ixs_arr) < 0):
            order = np.argsort(ixs_arr)
            adj = adj[order, :][:, order]
            dst = dst[order, :][:, order]
        return adj, dst


def _csr_from_rows(n: int, k: int, idx: np.ndarray, vals: np.ndarray, keep: np.ndarray | None = None) -> csr_matrix:
    """(n, k) row-major neighbour table with ascending indices per row -> canonical CSR (int32 indices / indptr)."""
    if keep is None:
        indptr = np.arange(0, n * k + 1, k, dtype=np.int32)
        m = csr_matrix((vals.reshape(-1), idx.reshape(-1), indptr), shape=(n, n))
    else:
        indptr = np.zeros(n + 1, dtype=np.int32)
        np.cumsum(keep.sum(axis=1), out=indptr[1:])
        m = csr_matrix((vals[keep], idx[keep], indptr), shape=(n, n))
    m.has_sorted_indices = True
    return m


class KNNBuilder(_Builder):
    """k-nearest-neighbour graph (``neighbors.py:157-209``): directed, ``n_neighs`` entries per row, float32 ones and float64
    euclidean distances."""

    def __init__(self, n_neighs: int = 6, transform=None, set_diag: bool = False, percentile: float | None = None, ctx: Context | None = None):
        assert_positive(n_neighs, name="n_neighs")
        super().__init__(transform, set_diag, percentile, ctx)
        self.n_neighs = n_neighs

    def uns_params(self) -> dict[str, Any]:
        return {"coord_type": CoordType.GENERIC.v, "n_neighbors": self.n_neighs, "transform": self.transform.v}

    def _device_args(self):
        return 0, int(self.n_neighs), 1, 0.0, None

    def build_graph(self, coords):
        dist, idx = knn_2d(coords, self.n_neighs, ctx=self.ctx)
        n = idx.shape[0]
        adj = _csr_from_rows(n, self.n_neighs, idx, np.ones(idx.shape, dtype=np.float32))
        dst = _csr_from_rows(n, self.n_neighs, idx, dist)
        self._diagonals(adj, dst)
        return adj, dst


class RadiusBuilder(_Builder):
    """Radius graph (``neighbors.py:212-270``); a tuple radius builds with the larger value and prunes to the interval."""

    def __init__(self, radius, transform=None, set_diag: bool = False, percentile: float | None = None, ctx: Context | None = None):
        super().__init__(transform, set_diag, percentile, ctx)
        self.radius = list(radius) if isinstance(radius, tuple) else radius

    def _interval(self):
        return tuple(sorted(self.radius)) if isinstance(self.radius, list) else None

    def uns_params(self) -> dict[str, Any]:
        return {"coord_type": CoordType.GENERIC.v, "radius": self.radius, "transform": self.transform.v}

    def _device_args(self):
        r = self.radius if isinstance(self.radius, int | float) else max(self.radius)
        return 2, 0, 1, r, self._interval()

    def build_graph(self, coords):
        r = self.radius if isinstance(self.radius, int | float) else max(self.radius)
        indptr, idx, dist = radius_2d(coords, r, ctx=self.ctx)
        n = indptr.size - 1
        ip = indptr.astype(np.int32)
        adj = csr_matrix((np.ones(idx.size, dtype=np.float32), idx, ip), shape=(n, n))
        dst = csr_matrix((dist, idx.copy(), ip.copy()), shape=(n, n))
        adj.has_sorted_indices = dst.has_sorted_indices = True
        self._diagonals(adj, dst)
        return adj, dst


class GridBuilder(_Builder):
    """Grid graph for Visium-like lattices (``neighbors.py:335-419``): ``n_neighs`` nearest candidates, those farther than
    1.3 x the median candidate distance dropped; ``n_rings > 1`` adds graph-distance shells (``dst`` holds the ring number)."""

    def __init__(self, n_neighs: int = 6, n_rings: int = 1, delaunay: bool = False, transform=None, set_diag: bool = False, ctx: Context | None = None):
        assert_positive(n_neighs, name="n_neighs")
        assert_positive(n_rings, name="n_rings")
        if delaunay:
            raise NotImplementedError("`delaunay=True` needs a Delaunay triangulation (Qhull); the GPU builders offer kNN, radius and grid graphs.")
        super().__init__(transform, set_diag, None, ctx)
        self.n_neighs, self.n_rings, self.delaunay = n_neighs, n_rings, delaunay

    def uns_params(self) -> dict[str, Any]:
        return {"coord_type": CoordType.GRID.v, "n_neighbors": self.n_neighs, "n_rings": self.n_rings, "delaunay": self.delaunay,
                "transform": self.transform.v}

    def _device_args(self):
        return 1, int(self.n_neighs), int(self.n_rings), 0.0, None

    def _base_adjacency(self, coords, *, set_diag: bool) -> csr_matrix:
        dist, idx, med = knn_2d(coords, self.n_neighs, median=True, ctx=self.ctx)
        keep = dist < med * 1.3  # neighbors.py:408-409
        adj = _csr_from_rows(idx.shape[0], self.n_neighs, idx, np.ones(idx.shape, dtype=np.float32), keep)
        if set_diag:
            adj.setdiag(1.0)
        return adj

    def build_graph(self, coords):
        if self.n_rings > 1:  # neighbors.py:372-386
            adj = self._base_adjacency(coords, set_diag=True)
            res, walk = adj, adj
            for i in range(self.n_rings - 1):
                walk = walk @ adj
                walk[res.nonzero()] = 0.0
                walk.eliminate_zeros()
                walk.data[:] = i + 2.0
                res = res + walk
            adj = res
            adj.setdiag(float(self.set_diag))
            adj.eliminate_zeros()
            dst = adj.copy()
            adj.data[:] = 1.0
        else:
            adj = self._base_adjacency(coords, set_diag=self.set_diag)
            dst = adj.copy()
        if self.set_diag or self.n_rings > 1:
            dst.setdiag(0.0)
        return adj, dst


class DelaunayBuilder(_Builder):
    """Delaunay graph (``neighbors.py:272-332``): the edges of the Delaunay triangulation, float32 ones and euclidean distances
    in the coordinates' dtype.  ``radius`` only prunes: a scalar ``r`` keeps edges of length in ``(0.0, r)``, a tuple is sorted
    and used as the interval, ``None`` keeps every edge."""

    def __init__(self, radius=None, transform=None, set_diag: bool = False, percentile: float | None = None, ctx: Context | None = None):
        if isinstance(radius, int | float):
            radius = (0.0, float(radius))
        super().__init__(transform, set_diag, percentile, ctx)
        self.radius = list(radius) if isinstance(radius, tuple) else radius

    def _interval(self):
        return None if self.radius is None else tuple(sorted(self.radius))

    def uns_params(self) -> dict[str, Any]:
        return {"coord_type": CoordType.GENERIC.v, "radius": self.radius, "transform": self.transform.v}

    def _device_args(self):
        return 3, 0, 1, 0.0, self._interval()

    def build_device(self, d: DevArray, device: int | None = None, libraries: tuple[np.ndarray, np.ndarray] | None = None):
        from scipy.spatial import QhullError

        try:
            return super().build_device(d, device, libraries)
        except ValueError as e:
            if str(e).startswith("QhullError"):
                raise QhullError(str(e)) from None
            raise

    def build_graph(self, coords):
        coords = np.asarray(coords)
        n = coords.shape[0]
        indptr, idx = delaunay_2d(coords, ctx=self.ctx)
        ip = indptr.astype(np.int32)
        adj = csr_matrix((np.ones(idx.size, dtype=np.float32), idx, ip), shape=(n, n))
        rows = np.repeat(np.arange(n), np.diff(indptr))
        dst = csr_matrix((np.linalg.norm(coords[rows] - coords[idx], axis=1), idx.copy(), ip.copy()), shape=(n, n))
        adj.has_sorted_indices = dst.has_sorted_indices = True
        self._diagonals(adj, dst)
        return adj, dst


# ---------------------------------------------------------------------------------------------------------
# public functions
# ---------------------------------------------------------------------------------------------------------
def _library_rows(adata, library_key: str | None) -> tuple[np.ndarray, np.ndarray] | None:
    """The observations of every library (the host path's ``np.where(codes == code)``) as (ptr int64, rows int32)."""
    if library_key is None:
        return None
    assert_categorical_obs(adata, key=library_key)
    codes = np.asarray(adata.obs[library_key].array.codes)
    n_libs = len(adata.obs[library_key].cat.categories)
    if n_libs == 0:
        raise ValueError(f"`adata.obs[{library_key!r}]` has no categories.")
    rows = np.argsort(codes, kind="stable").astype(np.int32)
    counts = np.bincount(codes[codes >= 0], minlength=n_libs)
    ptr = np.zeros(n_libs + 1, dtype=np.int64)
    np.cumsum(counts, out=ptr[1:])
    skip = int((codes < 0).sum())  # observations without a library belong to no block
    return ptr, np.ascontiguousarray(rows[skip:])


def _run(adata, builder: _Builder, *, spatial_key: str, library_key: str | None, key_added: str, copy: bool, device: int | None = None):
    """``_run_spatial_neighbors`` (``_build.py:789-850``)."""
    start = time.perf_counter()
    dev = _device_coords(adata.obsm[spatial_key])
    if dev is not None:
        adj, dst = builder.build_device(dev, device, _library_rows(adata, library_key))
    elif library_key is not None:
        assert_categorical_obs(adata, key=library_key)
        libs = adata.obs[library_key].cat.categories
        codes = np.asarray(adata.obs[library_key].array.codes)
        coords = np.asarray(adata.obsm[spatial_key])
        mats, idxs = [], []
        for code in range(len(libs)):
            idx = np.where(codes == code)[0]
            mats.append(builder.build(np.ascontiguousarray(coords[idx])))
            idxs.extend(idx.tolist())
        adj, dst = builder.combine(mats, idxs)
    else:
        adj, dst = builder.build(adata.obsm[spatial_key])
    logg.info("Creating graph using `%s` transform", builder.transform)
    neighs_key = Key.uns.spatial_neighs(key_added)
    conns_key = Key.obsp.spatial_conn(key_added)
    dists_key = Key.obsp.spatial_dist(key_added)
    if copy:
        return SpatialNeighborsResult(connectivities=adj, distances=dst)
    _save_data(adata, attr="obsp", key=conns_key, data=adj)
    _save_data(adata, attr="obsp", key=dists_key, data=dst, prefix=False)
    _save_data(adata, attr="uns", key=neighs_key, data={"connectivities_key": conns_key, "distances_key": dists_key, "params": builder.uns_params()},
               prefix=False, time_start=start)
    return None


def _host_context(adata, spatial_key: str, device: int | None) -> Context | None:
    """The context of the host path; device coordinates are built on their own device (``_Builder.build_device``)."""
    return None if _device_coords(adata.obsm[spatial_key]) is not None else default_context(device)


def _prepare(data, spatial_key, table_key):
    adata = extract_adata_if_sdata(data, table_key=table_key)
    assert_spatial_basis(adata, spatial_key)
    return adata


def spatial_neighbors_knn(data: Any, *, spatial_key: str = Key.obsm.spatial, elements_to_coordinate_systems: dict[str, str] | None = None,
                          table_key: str | None = None, library_key: str | None = None, n_neighs: int = 6, percentile: float | None = None,
                          transform=None, set_diag: bool = False, key_added: str = "spatial", copy: bool = False, n_jobs: int = 1,
                          device: int | None = None) -> SpatialNeighborsResult | None:
    """k-nearest-neighbour graph from spatial coordinates (``_build.py:484-549``); ``n_jobs`` is accepted and ignored."""
    adata = _prepare(data, spatial_key, table_key)
    builder = KNNBuilder(n_neighs=n_neighs, percentile=percentile, transform=transform, set_diag=set_diag, ctx=_host_context(adata, spatial_key, device))
    return _run(adata, builder, spatial_key=spatial_key, library_key=library_key, key_added=key_added, copy=copy,
                device=device)


def spatial_neighbors_radius(data: Any, *, spatial_key: str = Key.obsm.spatial, elements_to_coordinate_systems: dict[str, str] | None = None,
                             table_key: str | None = None, library_key: str | None = None, radius: float | tuple[float, float] = 1.0,
                             percentile: float | None = None, transform=None, set_diag: bool = False, key_added: str = "spatial",
                             copy: bool = False, n_jobs: int = 1, device: int | None = None) -> SpatialNeighborsResult | None:
    """Radius graph from spatial coordinates (``_build.py:553-620``)."""
    adata = _prepare(data, spatial_key, table_key)
    builder = RadiusBuilder(radius=radius, percentile=percentile, transform=transform, set_diag=set_diag, ctx=_host_context(adata, spatial_key, device))
    return _run(adata, builder, spatial_key=spatial_key, library_key=library_key, key_added=key_added, copy=copy,
                device=device)


def spatial_neighbors_grid(data: Any, *, spatial_key: str = Key.obsm.spatial, elements_to_coordinate_systems: dict[str, str] | None = None,
                           table_key: str | None = None, library_key: str | None = None, n_neighs: int = 6, n_rings: int = 1,
                           delaunay: bool = False, transform=None, set_diag: bool = False, key_added: str = "spatial", copy: bool = False,
                           n_jobs: int = 1, device: int | None = None) -> SpatialNeighborsResult | None:
    """Grid graph for Visium-like coordinates (``_build.py:701-786``)."""
    assert_positive(n_rings, name="n_rings")
    assert_positive(n_neighs, name="n_neighs")
    adata = _prepare(data, spatial_key, table_key)
    builder = GridBuilder(n_neighs=n_neighs, n_rings=n_rings, delaunay=delaunay, transform=transform, set_diag=set_diag,
                          ctx=_host_context(adata, spatial_key, device))
    return _run(adata, builder, spatial_key=spatial_key, library_key=library_key, key_added=key_added, copy=copy,
                device=device)


def spatial_neighbors_delaunay(data: Any, *, spatial_key: str = Key.obsm.spatial, elements_to_coordinate_systems: dict[str, str] | None = None,
                               table_key: str | None = None, library_key: str | None = None, radius: float | tuple[float, float] | None = None,
                               percentile: float | None = None, transform=None, set_diag: bool = False, key_added: str = "spatial",
                               copy: bool = False, n_jobs: int = 1, device: int | None = None) -> SpatialNeighborsResult | None:
    """Delaunay graph from spatial coordinates (``_build.py:625-697``); ``n_jobs`` is accepted and ignored."""
    adata = _prepare(data, spatial_key, table_key)
    builder = DelaunayBuilder(radius=radius, percentile=percentile, transform=transform, set_diag=set_diag, ctx=_host_context(adata, spatial_key, device))
    return _run(adata, builder, spatial_key=spatial_key, library_key=library_key, key_added=key_added, copy=copy, device=device)


def spatial_neighbors_from_builder(data: Any, builder: _Builder, *, spatial_key: str = Key.obsm.spatial,
                                   elements_to_coordinate_systems: dict[str, str] | None = None, table_key: str | None = None,
                                   library_key: str | None = None, key_added: str = "spatial", copy: bool = False, n_jobs: int = 1,
                                   device: int | None = None) -> SpatialNeighborsResult | None:
    """Spatial graph from a builder the caller constructed (``_build.py:388-460``): any of ``KNNBuilder``, ``RadiusBuilder``,
    ``GridBuilder`` and ``DelaunayBuilder``."""
    if not isinstance(builder, _Builder):
        raise TypeError(f"Expected a graph builder, found `{type(builder).__name__}`.")
    adata = _prepare(data, spatial_key, table_key)
    if builder.ctx is None and _device_coords(adata.obsm[spatial_key]) is None:
        import copy as _copy

        builder = _copy.copy(builder)  # the caller's builder keeps no context of this call
        builder.ctx = default_context(device)
    return _run(adata, builder, spatial_key=spatial_key, library_key=library_key, key_added=key_added, copy=copy, device=device)
