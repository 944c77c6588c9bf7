"""The graph builder contract and the post-processors of ``squidpy.gr.neighbors`` (``src/squidpy/gr/neighbors.py``:
``GraphBuilder`` / ``GraphBuilderCSR`` :54-156, ``DistanceIntervalPostprocessor`` / ``PercentilePostprocessor`` /
``TransformPostprocessor`` :423-477).

A custom builder fed device coordinates naturally returns a device graph, such as the torch ``sparse_csr`` CUDA tensors the
built-in builders export.  The post-processors and ``GraphBuilderCSR.combine`` therefore take both kinds of graph: scipy CSRs
are processed on the host with the reference's scipy steps, and CSRs in GPU memory (torch ``sparse_csr`` or cupyx-style, int32
or int64 indices, ascending columns) on their GPU (``sqb_graph_postprocess`` / ``sqb_graph_combine``), which returns torch
``sparse_csr`` CUDA tensors equal to the host result after ``sort_indices()``: the same stored entries, explicit zeros included,
and the same values and dtypes.
"""

from __future__ import annotations

import ctypes as C
import math
import warnings
from abc import ABC, abstractmethod
from collections.abc import Callable, Sequence
from dataclasses import dataclass
from typing import Any, TypeVar

import numpy as np
from scipy.sparse import SparseEfficiencyWarning, block_diag, csr_matrix

from .._constants import Transform
from .._device import DevSparse, _torch_stream, array_device, common_stream, device_graph, sparse_args
from .._lib import check, default_context, load, pointer_device

__all__ = ["GraphMatrixT", "GraphPostprocessor", "GraphBuilder", "GraphBuilderCSR", "DistanceIntervalPostprocessor", "PercentilePostprocessor",
           "TransformPostprocessor"]

GraphMatrixT = TypeVar("GraphMatrixT")
GraphPostprocessor = Callable[[GraphMatrixT, GraphMatrixT], tuple[GraphMatrixT, GraphMatrixT]]
CoordT = TypeVar("CoordT")

_TRANSFORM_CODES = {Transform.NONE: 0, Transform.SPECTRAL: 1, Transform.COSINE: 2}


# ---------------------------------------------------------------------------------------------------------
# host steps (scipy; follow neighbors.py:427-477)
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
    """D^-1/2 A D^-1/2 with D = column sums (``symmetric_normalize_csr``, neighbors.py:514-540), float32 result."""
    if not a.nnz:
        return a
    degrees = np.squeeze(np.array(np.sqrt(1.0 / a.sum(axis=0))))
    rows = np.repeat(np.arange(a.shape[0]), np.diff(a.indptr))
    res = (degrees[rows] * degrees[a.indices] * a.data).astype(np.float32)
    return csr_matrix((res, a.indices, a.indptr), shape=a.shape)


def _apply_transform(adj: csr_matrix, dst: csr_matrix, transform: Transform) -> tuple[csr_matrix, csr_matrix]:
    # eliminate_zeros() of the reference (neighbors.py:466-467); a full pass only when there is something to drop
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
# device graphs
# ---------------------------------------------------------------------------------------------------------
def graph_pair_device(adj: Any, dst: Any) -> int | None:
    """The CUDA device holding both matrices of a graph, or ``None`` when both are host objects.  One on the host and the other
    on a GPU, or the two on different GPUs, raise ``TypeError``."""
    da, dd = device_graph(adj), device_graph(dst)
    if da is None and dd is None:
        return None
    if da is None or dd is None:
        raise TypeError("The connectivities and the distances must both be on the host or both on the same GPU; found one on the host "
                        "and the other on a GPU.")
    on_a, on_d = array_device(da, pointer_device), array_device(dd, pointer_device)
    if on_a != on_d:
        raise TypeError(f"The connectivities (cuda:{on_a}) and the distances (cuda:{on_d}) must be on the same GPU.")
    return on_a


def _device_csr(d: DevSparse, n: int, what: str, dtypes: tuple[type, ...]) -> tuple[int, int, int, int, int, int]:
    """(nnz, indptr, indptr_bits, indices, index_bits, data) of an n x n device CSR with values of one of ``dtypes``."""
    if d.format != "csr":
        raise NotImplementedError(f"The {what} must be a CSR matrix on the GPU, found `{d.format}`.")
    if tuple(d.shape) != (n, n):
        raise ValueError(f"Expected the {what} to be of shape `{(n, n)}`, found `{tuple(d.shape)}`.")
    if d.data.dtype not in tuple(np.dtype(t) for t in dtypes):
        names = " or ".join(np.dtype(t).name for t in dtypes)
        raise TypeError(f"The {what} must hold {names} values on the GPU, found `{d.data.dtype}`.")
    ip_bits, ix_bits, nnz = sparse_args(d, n)
    v = d.data
    if len(v.shape) != 1 or v.shape[0] != nnz or (nnz > 1 and v.strides[0] != 1):
        raise ValueError(f"The {what}' values must be a contiguous 1-D array of `{nnz}` entries.")
    return nnz, d.indptr.ptr, ip_bits, d.indices.ptr or 0, ix_bits, v.ptr or 0


def _pair(adj: Any, dst: Any) -> tuple[int, DevSparse, DevSparse, int]:
    on = graph_pair_device(adj, dst)
    da, dd = device_graph(adj), device_graph(dst)
    if tuple(da.shape) != tuple(dd.shape) or da.shape[0] != da.shape[1]:
        raise ValueError(f"Expected square connectivities and distances of one shape, found `{tuple(da.shape)}` and `{tuple(dd.shape)}`.")
    streams = {s for s in (common_stream(da), common_stream(dd)) if s}
    if len(streams) > 1:
        raise ValueError(f"The connectivities and the distances name different producer streams: {sorted(streams)}.")
    return on, da, dd, streams.pop() if streams else 0


def export_graph(h: C.c_void_p, on: int, n: int, nnz_a: int, nnz_d: int, f64: bool):
    """The graph of a ``sqb_graph`` handle as torch ``sparse_csr`` CUDA tensors on device ``on`` (int32 indices); frees the handle."""
    import torch

    lib = load()
    try:
        dev = torch.device("cuda", on)
        parts = [torch.empty(n + 1, dtype=torch.int32, device=dev), torch.empty(nnz_a, dtype=torch.int32, device=dev),
                 torch.empty(nnz_a, dtype=torch.float32, device=dev), torch.empty(n + 1, dtype=torch.int32, device=dev),
                 torch.empty(nnz_d, dtype=torch.int32, device=dev), torch.empty(nnz_d, dtype=torch.float64 if f64 else torch.float32, device=dev)]
        check(lib.sqb_graph_export(h, *(t.data_ptr() or None for t in parts), _torch_stream(parts[0])))
    finally:
        lib.sqb_graph_free(h)
    adj = torch.sparse_csr_tensor(parts[0], parts[1], parts[2], size=(n, n))
    dst = torch.sparse_csr_tensor(parts[3], parts[4], parts[5], size=(n, n))
    return adj, dst


def _postprocess_device(adj: Any, dst: Any, op: int, a: float = 0.0, b: float = 0.0, transform: int = 0):
    """One post-processor (op 0 interval [a, b], 1 percentile a, 2 transform) of a device graph on its GPU."""
    on, da, dd, stream = _pair(adj, dst)
    n = int(da.shape[0])
    A = _device_csr(da, n, "connectivities", (np.float32,))
    D = _device_csr(dd, n, "distances", (np.float32, np.float64))
    f64 = dd.data.dtype == np.float64
    ctx = default_context(on)
    h, nnz_a, nnz_d, f64_out = C.c_void_p(), C.c_int64(), C.c_int64(), C.c_int()
    with ctx.lock:
        check(load().sqb_graph_postprocess(ctx.handle, n, A[0], A[1], A[2], A[3] or None, A[4], A[5] or None, D[0], D[1], D[2], D[3] or None, D[4],
                                           D[5] or None, int(f64), stream, op, float(a), float(b), transform, C.byref(h), C.byref(nnz_a),
                                           C.byref(nnz_d), C.byref(f64_out)))
        return export_graph(h, on, n, nnz_a.value, nnz_d.value, bool(f64_out.value))


def _combine_device(mats: Sequence[tuple[Any, Any]], ixs: Sequence[int]):
    """``GraphBuilderCSR.combine`` of device blocks on their GPU."""
    ons, descs_a, descs_d, sizes, streams, dtypes = set(), [], [], [], set(), set()
    for adj, dst in mats:
        on, da, dd, stream = _pair(adj, dst)
        n = int(da.shape[0])
        ons.add(on)
        streams.add(stream)
        descs_a.append(_device_csr(da, n, "connectivities", (np.float32,)))
        descs_d.append(_device_csr(dd, n, "distances", (np.float32, np.float64)))
        dtypes.add(dd.data.dtype)
        sizes.append(n)
    if len(ons) > 1:
        raise TypeError(f"The library graphs must all be on one GPU, found {sorted(ons)}.")
    if len(dtypes) > 1:
        raise TypeError(f"The library graphs' distances must share one dtype, found {sorted(str(d) for d in dtypes)}.")
    streams.discard(0)
    if len(streams) > 1:
        raise ValueError(f"The library graphs name different producer streams: {sorted(streams)}.")
    ix = np.asarray(ixs, dtype=np.int64).reshape(-1)
    if ix.size != sum(sizes):
        raise ValueError(f"Expected {sum(sizes)} observation indices for the library graphs, found {ix.size}.")
    if np.unique(ix).size != ix.size:
        raise ValueError("The observation indices of the library graphs must be distinct.")
    out_row = np.empty(ix.size, dtype=np.int32)
    out_row[np.argsort(ix, kind="stable")] = np.arange(ix.size, dtype=np.int32)  # the rank of every observation
    on = ons.pop()
    ctx = default_context(on)
    block_n = np.asarray(sizes, dtype=np.int64)
    a_desc = np.asarray(descs_a, dtype=np.int64).reshape(-1)
    d_desc = np.asarray(descs_d, dtype=np.int64).reshape(-1)
    f64 = dtypes.pop() == np.float64
    h, n_out, nnz_a, nnz_d, f64_out = C.c_void_p(), C.c_int64(), C.c_int64(), C.c_int64(), C.c_int()
    with ctx.lock:
        check(load().sqb_graph_combine(ctx.handle, len(sizes), block_n.ctypes.data, a_desc.ctypes.data, d_desc.ctypes.data, int(f64),
                                       streams.pop() if streams else 0, out_row.ctypes.data, C.byref(h), C.byref(n_out), C.byref(nnz_a),
                                       C.byref(nnz_d), C.byref(f64_out)))
        return export_graph(h, on, n_out.value, nnz_a.value, nnz_d.value, bool(f64_out.value))


# ---------------------------------------------------------------------------------------------------------
# post-processors (neighbors.py:441-477)
# ---------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class DistanceIntervalPostprocessor:
    """Keep the entries whose distance lies in ``interval`` (``[min, max]``): the others become explicit zeros in both
    matrices, by position, and the connectivities keep their diagonal."""

    interval: tuple[float, float]

    def __call__(self, adj, dst):
        if graph_pair_device(adj, dst) is not None:
            minn, maxx = self.interval
            if device_graph(adj).indices.shape[0] != device_graph(dst).indices.shape[0]:
                raise IndexError(f"boolean index did not match indexed array along axis 0; size of axis is {device_graph(adj).indices.shape[0]} "
                                 f"but size of corresponding boolean axis is {device_graph(dst).indices.shape[0]}")
            return _postprocess_device(adj, dst, 0, float(minn), float(maxx))
        _filter_by_radius_interval(adj, dst, self.interval)
        return adj, dst


@dataclass(frozen=True)
class PercentilePostprocessor:
    """Zero the connectivities and distances of the entries whose distance exceeds ``np.percentile(dst.data, percentile)``."""

    percentile: float

    def __call__(self, adj, dst):
        if graph_pair_device(adj, dst) is not None:
            if not 0.0 <= float(self.percentile) <= 100.0 or math.isnan(float(self.percentile)):
                raise ValueError("Percentiles must be in the range [0, 100]")
            if device_graph(dst).indices.shape[0] == 0:
                raise IndexError("index -1 is out of bounds for axis 0 with size 0")
            return _postprocess_device(adj, dst, 1, float(self.percentile))
        return _percentile(adj, dst, self.percentile)


@dataclass(frozen=True)
class TransformPostprocessor:
    """``eliminate_zeros`` on both matrices, then the ``transform`` (none, spectral, cosine) of the connectivities."""

    transform: Transform

    def __call__(self, adj, dst):
        if graph_pair_device(adj, dst) is not None:
            return _postprocess_device(adj, dst, 2, transform=_TRANSFORM_CODES[Transform(self.transform)])
        return _apply_transform(adj, dst, Transform(self.transform))


# ---------------------------------------------------------------------------------------------------------
# builders (neighbors.py:54-156)
# ---------------------------------------------------------------------------------------------------------
class GraphBuilder[CoordT, GraphMatrixT](ABC):
    """Base class of spatial graph construction strategies.

    Custom builders implement :meth:`build_graph` and :meth:`uns_params`; :meth:`postprocessors` and :meth:`combine` may be
    overridden.  Post-processors can also be passed to ``__init__``."""

    def __init__(self, transform: str | Transform | None = None, set_diag: bool = False, percentile: float | None = None,
                 postprocessors: Sequence[GraphPostprocessor] = ()) -> None:
        self.transform = Transform.NONE if transform is None else Transform(transform)
        self.set_diag = set_diag
        self.percentile = percentile
        self._postprocessors: list[GraphPostprocessor] = list(postprocessors)

    def build(self, coords):
        adj, dst = self.build_graph(coords)
        for postprocessor in self.postprocessors():
            adj, dst = postprocessor(adj, dst)
        return adj, dst

    @abstractmethod
    def build_graph(self, coords):
        """Construct raw adjacency and distance matrices."""

    def postprocessors(self) -> Sequence[GraphPostprocessor]:
        """Return post-build processing steps for ``(adj, dst)``."""
        return self._postprocessors

    @abstractmethod
    def uns_params(self) -> dict[str, Any]:
        """Parameters stored in ``adata.uns`` after graph construction (values :mod:`anndata` can write, e.g. no tuples)."""

    def combine(self, mats, ixs):
        """Combine per-library results into a single graph; override to support ``library_key``."""
        raise NotImplementedError("Using `library_key` with this graph builder is not implemented yet.")


class GraphBuilderCSR(GraphBuilder[Any, csr_matrix], ABC):
    """CSR-based graph construction strategy: ``build`` suppresses ``SparseEfficiencyWarning`` and ``combine`` joins the
    per-library graphs.  Graphs may be scipy CSRs or CSRs in GPU memory; device graphs are post-processed and combined on
    their GPU."""

    def build(self, coords):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", SparseEfficiencyWarning)
            return super().build(coords)

    @abstractmethod
    def build_graph(self, coords):
        """Construct raw adjacency and distance matrices."""

    def combine(self, mats, ixs):
        """Per-library blocks -> one graph in the original observation order (``neighbors.py:137-154``)."""
        mats = list(mats)
        places = {graph_pair_device(a, d) is not None for a, d in mats}
        if places == {True}:
            return _combine_device(mats, ixs)
        if len(places) > 1:
            raise TypeError("The library graphs must all be on the host or all on a GPU.")
        adj = block_diag([m[0] for m in mats], format="csr")
        dst = block_diag([m[1] for m in mats], format="csr")
        ixs_arr = np.asarray(ixs)
        if ixs_arr.size and np.any(np.diff(ixs_arr) < 0):
            order = np.argsort(ixs_arr)
            adj = adj[order, :][:, order]
            dst = dst[order, :][:, order]
        return adj, dst
