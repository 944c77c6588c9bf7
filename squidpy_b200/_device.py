"""Device-resident feature matrices: what ``AutocorrPlan.load`` / ``spatial_autocorr`` accept besides numpy and scipy.

* dense objects exposing ``__cuda_array_interface__`` (cupy, numba, torch CUDA tensors);
* sparse objects in the cupyx style (``.format`` in {csr, csc}, ``.indptr`` / ``.indices`` / ``.data`` exposing the
  interface, ``.shape``) and torch ``sparse_csr`` / ``sparse_csc`` CUDA tensors.

Nothing here imports cupy, and torch only when the object is already a torch tensor.  The arrays are described by their
device pointers and handed to the C ABI (``sqb_autocorr_load_*_device``); they are never read on the host.
"""

from __future__ import annotations

import sys
from dataclasses import dataclass
from typing import Any

import numpy as np

SPARSE_FORMATS = ("csr", "csc")
# dtype code of sqb_autocorr_load_*_device: float32 stays float32, the others become float64 on the device
DTYPE_CODES = {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.float16): 2, np.dtype(np.int32): 3, np.dtype(np.int64): 4}


@dataclass
class DevArray:
    """One array described by the CUDA Array Interface; strides in elements, ``stream`` as in CAI v3 (0 = none)."""

    ptr: int
    shape: tuple[int, ...]
    dtype: np.dtype
    strides: tuple[int, ...]
    stream: int
    owner: Any  # keeps the exporting object alive while the pointer is in use


@dataclass
class DevSparse:
    """A device CSR or CSC matrix of ``shape``."""

    format: str
    shape: tuple[int, int]
    indptr: DevArray
    indices: DevArray
    data: DevArray

    @property
    def arrays(self) -> tuple[DevArray, DevArray, DevArray]:
        return self.indptr, self.indices, self.data


def parse_cai(obj: Any, stream: int | None = None) -> DevArray:
    """Parse ``obj.__cuda_array_interface__`` (versions 0-3).  ``stream`` overrides the interface's own ``stream``
    (torch reports version 2, without one: its current stream is passed instead)."""
    d = obj.__cuda_array_interface__
    version = int(d.get("version", 0))
    if not 0 <= version <= 3:
        raise ValueError(f"Unsupported __cuda_array_interface__ version `{version}`.")
    if d.get("mask") is not None:
        raise ValueError("Masked device arrays (`__cuda_array_interface__['mask']`) are not supported.")
    shape = tuple(int(s) for s in d["shape"])
    dtype = np.dtype(d["typestr"])
    if dtype.byteorder == ">":
        raise ValueError(f"Big-endian device arrays (`{d['typestr']}`) are not supported.")
    ptr = int(d["data"][0] or 0)
    if d.get("strides") is None:
        strides, step = [], 1
        for s in reversed(shape):
            strides.append(step)
            step *= max(s, 1)
        strides = tuple(reversed(strides))
    else:
        if any(int(s) % dtype.itemsize for s in d["strides"]):
            raise ValueError(f"Strides `{d['strides']}` are not multiples of the item size {dtype.itemsize}.")
        strides = tuple(int(s) // dtype.itemsize for s in d["strides"])
    if stream is None:
        stream = d.get("stream") if version >= 3 else None
        if stream == 0:
            raise ValueError("`__cuda_array_interface__['stream'] = 0` is ambiguous and not allowed (use 1 for the legacy default stream).")
        stream = 0 if stream is None else int(stream)
    return DevArray(ptr, shape, dtype, strides, int(stream), obj)


def _torch_stream(t: Any) -> int:
    """CAI stream value of torch's current stream on the tensor's device (its NULL stream is the legacy default: 1)."""
    torch = sys.modules["torch"]
    s = torch.cuda.current_stream(t.device).cuda_stream
    return int(s) if s else 1


def device_matrix(m: Any) -> DevArray | DevSparse | None:
    """The device description of ``m``, or ``None`` when ``m`` is a host object (numpy, scipy, a CPU tensor)."""
    torch = sys.modules.get("torch")
    if torch is not None and isinstance(m, torch.Tensor):
        if m.layout == torch.strided:
            return parse_cai(m.detach(), stream=_torch_stream(m)) if m.is_cuda else None
        if m.layout == torch.sparse_csr:
            fmt, parts = "csr", (m.crow_indices(), m.col_indices(), m.values())
        elif m.layout == torch.sparse_csc:
            fmt, parts = "csc", (m.ccol_indices(), m.row_indices(), m.values())
        else:
            raise NotImplementedError(f"Sparse layout `{m.layout}` is not supported; supported formats: {', '.join(SPARSE_FORMATS)}.")
        if not m.is_cuda:
            return None
        st = _torch_stream(m)
        ip, ix, dv = (parse_cai(p.detach(), stream=st) for p in parts)
        return DevSparse(fmt, (int(m.shape[0]), int(m.shape[1])), ip, ix, dv)
    fmt = getattr(m, "format", None)
    if isinstance(fmt, str) and hasattr(getattr(m, "data", None), "__cuda_array_interface__"):
        if fmt not in SPARSE_FORMATS:
            raise NotImplementedError(f"Sparse format `{fmt}` is not supported; supported formats: {', '.join(SPARSE_FORMATS)}.")
        ip, ix, dv = parse_cai(m.indptr), parse_cai(m.indices), parse_cai(m.data)
        return DevSparse(fmt, (int(m.shape[0]), int(m.shape[1])), ip, ix, dv)
    if hasattr(m, "__cuda_array_interface__"):
        return parse_cai(m)
    return None


def common_stream(d: DevArray | DevSparse) -> int:
    """The one producer stream of a (sparse) device matrix; its arrays must not name different streams."""
    arrays = d.arrays if isinstance(d, DevSparse) else (d,)
    streams = {a.stream for a in arrays if a.stream != 0}
    if len(streams) > 1:
        raise ValueError(f"The arrays of the sparse matrix name different producer streams: {sorted(streams)}.")
    return streams.pop() if streams else 0


def array_device(d: DevArray | DevSparse, pointer_device) -> int:
    """CUDA device holding every array of ``d`` (``pointer_device(ptr) -> ordinal or -1`` asks the driver).  Host memory
    presented through the interface, or arrays on different devices, raise ``ValueError``."""
    arrays = d.arrays if isinstance(d, DevSparse) else (d,)
    devices = set()
    for a in arrays:
        if a.ptr == 0:  # an empty array has no allocation
            continue
        dev = int(pointer_device(a.ptr))
        if dev < 0:
            raise ValueError("An array exposing `__cuda_array_interface__` points to host memory; pass it as a numpy / scipy object instead.")
        devices.add(dev)
    if not devices:
        raise ValueError("The device matrix has no allocated array.")
    if len(devices) > 1:
        raise ValueError(f"The arrays of the matrix live on different devices: {sorted(devices)}.")
    return devices.pop()


def dtype_code(a: DevArray) -> int:
    code = DTYPE_CODES.get(a.dtype)
    if code is None:
        raise TypeError(f"Device arrays of dtype `{a.dtype}` are not supported; use float32, float64, float16, int32 or int64.")
    return code


def index_bits(a: DevArray, what: str) -> int:
    if a.dtype not in (np.dtype(np.int32), np.dtype(np.int64)):
        raise TypeError(f"`{what}` must be int32 or int64, found `{a.dtype}`.")
    if len(a.shape) != 1 or (a.shape[0] > 1 and a.strides[0] != 1):
        raise ValueError(f"`{what}` must be a contiguous 1-D array.")
    return 8 * a.dtype.itemsize


def sparse_args(d: DevSparse, major: int) -> tuple[int, int, int]:
    """``(indptr_bits, index_bits, nnz)`` of a device CSR / CSC with ``major`` rows (columns for CSC), once its index arrays
    are int32 / int64 and contiguous and ``indptr`` has ``major + 1`` entries."""
    ip_bits, ix_bits = index_bits(d.indptr, "indptr"), index_bits(d.indices, "indices")
    if d.indptr.shape[0] != major + 1:
        raise ValueError(f"Expected `indptr` of length `{major + 1}`, found `{d.indptr.shape[0]}`.")
    return ip_bits, ix_bits, int(d.indices.shape[0])


@dataclass
class DevGraph:
    """The ABI arguments of a device neighbour graph (``sqb_nhood_create_device`` / ``sqb_interaction_matrix_device``).

    The arrays are handed over as given.  For a CSC graph they are the CSR of the transpose, so every C x C result computed
    from them is the transpose of the graph's: ``transposed`` tells the caller to transpose it back."""

    sparse: DevSparse
    n: int
    nnz: int
    indptr_bits: int
    index_bits: int
    transposed: bool
    stream: int

    @property
    def indptr(self) -> int:
        return self.sparse.indptr.ptr

    @property
    def indices(self) -> int:
        return self.sparse.indices.ptr


def device_graph(m: Any) -> DevSparse | None:
    """The device description of a neighbour graph (``obsp[key]``), or ``None`` for a host graph.  Graphs are sparse: a
    dense device array raises ``NotImplementedError``."""
    d = device_matrix(m)
    if isinstance(d, DevArray):
        raise NotImplementedError(f"Dense device graphs are not supported; supported formats: {', '.join(SPARSE_FORMATS)}.")
    return d


def graph_args(d: DevSparse, n_obs: int) -> DevGraph:
    """Check that ``d`` is an ``n_obs x n_obs`` graph with int32 / int64 index arrays and describe it for the C ABI."""
    if tuple(d.shape) != (n_obs, n_obs):
        raise ValueError(f"Expected the connectivity graph to be of shape `{(n_obs, n_obs)}`, found `{tuple(d.shape)}`.")
    ip_bits, ix_bits, nnz = sparse_args(d, n_obs)
    return DevGraph(d, n_obs, nnz, ip_bits, ix_bits, d.format == "csc", common_stream(d))


def _contiguous_1d(a: DevArray, size: int | None = None) -> bool:
    return len(a.shape) == 1 and (size is None or a.shape[0] == size) and (a.shape[0] <= 1 or a.strides[0] == 1)


def weight_graph_args(d: DevArray | DevSparse | None, n_obs: int) -> DevGraph | None:
    """The ``DevGraph`` of a device weight matrix that ``sqb_autocorr_create_device`` reads in place: an ``n_obs x n_obs`` CSR
    with contiguous int32 / int64 ``indptr`` (``n_obs + 1`` entries) and ``indices``, and a contiguous float32 / float64 ``data``
    of exactly as many entries.  ``None`` for anything else (host, dense or CSC matrices, other dtypes, strided or mis-sized
    arrays): spatial_autocorr then copies the matrix to the host as it does for every other weight matrix."""
    if not isinstance(d, DevSparse) or d.format != "csr" or tuple(d.shape) != (n_obs, n_obs):
        return None
    ints = (np.dtype(np.int32), np.dtype(np.int64))
    if d.indptr.dtype not in ints or d.indices.dtype not in ints or d.data.dtype not in (np.dtype(np.float32), np.dtype(np.float64)):
        return None
    nnz = d.indices.shape[0] if len(d.indices.shape) == 1 else -1
    if not (_contiguous_1d(d.indptr, n_obs + 1) and _contiguous_1d(d.indices) and _contiguous_1d(d.data, nnz)):
        return None
    return graph_args(d, n_obs)


# value dtype code of sqb_interaction_matrix_device: the autocorr codes plus bool (one byte per value)
GRAPH_VALUE_CODES = {**DTYPE_CODES, np.dtype(np.bool_): 5}


def graph_value_code(a: DevArray, nnz: int) -> int:
    code = GRAPH_VALUE_CODES.get(a.dtype)
    if code is None:
        raise TypeError(f"Device graph values of dtype `{a.dtype}` are not supported; use float32, float64, float16, int32, int64 or bool.")
    if len(a.shape) != 1 or a.shape[0] != nnz or (nnz > 1 and a.strides[0] != 1):
        raise ValueError(f"The graph's values must be a contiguous 1-D array of `{nnz}` entries.")
    return code


def feature_map(n_cols: int, positions: Any, lo: int = 0, hi: int | None = None) -> tuple[np.ndarray, int, np.ndarray]:
    """``col_map`` of ``sqb_autocorr_load_*_device`` for the selected features ``positions[lo:hi]`` (input feature of every
    selected feature, in output order; duplicates allowed).  Every distinct feature is loaded once, in order of first
    occurrence.  Returns ``(col_map int32[n_cols], n_out, expand)``: the scores of the shard are ``loaded_scores[expand]``."""
    pos = np.asarray(positions, dtype=np.int64).reshape(-1)[lo:hi]
    if pos.size and (pos.min() < 0 or pos.max() >= n_cols):
        raise IndexError(f"Feature indices must lie in [0, {n_cols}).")
    uniq, first, inverse = np.unique(pos, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty(order.size, dtype=np.int64)
    rank[order] = np.arange(order.size)
    col_map = np.full(n_cols, -1, dtype=np.int32)
    col_map[uniq] = rank
    return col_map, int(uniq.size), rank[inverse.reshape(-1)]


@dataclass
class DevMatrix:
    """The ABI arguments of a device expression matrix for ``sqb_dense_gather_device`` (observations x genes).

    ``format`` 0 dense (``x`` the array, ``strides`` in elements), 1 CSR, 2 CSC (``x`` the values); ``code`` the value dtype
    code (``DTYPE_CODES``)."""

    format: int
    shape: tuple[int, int]
    x: int
    indptr: int
    indptr_bits: int
    indices: int
    index_bits: int
    nnz: int
    dtype: np.dtype
    code: int
    strides: tuple[int, int]
    stream: int
    source: DevArray | DevSparse


def matrix_args(d: DevArray | DevSparse, shape: tuple[int, int]) -> DevMatrix:
    """Check that ``d`` is an expression matrix of ``shape`` in a supported layout and dtype, and describe it."""
    shape = (int(shape[0]), int(shape[1]))
    if tuple(d.shape) != shape:
        raise ValueError(f"Expected the expression matrix to be of shape `{shape}`, found `{tuple(d.shape)}`.")
    stream = common_stream(d)
    if isinstance(d, DevSparse):
        ip_bits, ix_bits, nnz = sparse_args(d, shape[0] if d.format == "csr" else shape[1])
        code = dtype_code(d.data)
        if len(d.data.shape) != 1 or d.data.shape[0] < nnz or (nnz > 1 and d.data.strides[0] != 1):
            raise ValueError(f"The matrix's values must be a contiguous 1-D array of `{nnz}` entries.")
        return DevMatrix(1 if d.format == "csr" else 2, shape, d.data.ptr, d.indptr.ptr, ip_bits, d.indices.ptr, ix_bits, nnz, d.data.dtype,
                         code, (0, 0), stream, d)
    if len(d.shape) != 2:
        raise ValueError(f"Expected a 2-D device array, found shape `{d.shape}`.")
    return DevMatrix(0, shape, d.ptr, 0, 32, 0, 32, 0, d.dtype, dtype_code(d), (int(d.strides[0]), int(d.strides[1])), stream, d)


def _host_array(a: Any) -> np.ndarray:
    torch = sys.modules.get("torch")
    if torch is not None and isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy()
    if hasattr(a, "get"):  # cupy
        return np.asarray(a.get())
    import torch  # any other exporter of the interface

    return torch.as_tensor(a, device="cuda").cpu().numpy()


def on_host(m: Any) -> Any:
    """``m`` itself when it is a host object, else its host copy (``to_host_matrix``): for the readers of ``obsm`` / ``obsp``
    that stage small arrays (coordinates, a neighbour graph) on the host anyway."""
    return m if device_matrix(m) is None else to_host_matrix(m)


def to_host_matrix(m: Any) -> Any:
    """Host copy of a device-resident matrix (numpy for dense, scipy CSR / CSC for sparse): for the weight matrix, which is
    small next to X and whose moments, S0 and row normalisation are computed on the host."""
    import scipy.sparse as sp

    d = device_matrix(m)
    if isinstance(d, DevArray):
        return _host_array(m)
    torch = sys.modules.get("torch")
    if torch is not None and isinstance(m, torch.Tensor):
        c = m.detach().cpu()
        if d.format == "csr":
            parts = (c.values().numpy(), c.col_indices().numpy(), c.crow_indices().numpy())
        else:
            parts = (c.values().numpy(), c.row_indices().numpy(), c.ccol_indices().numpy())
    else:
        parts = (_host_array(m.data), _host_array(m.indices), _host_array(m.indptr))
    return (sp.csr_matrix if d.format == "csr" else sp.csc_matrix)(parts, shape=d.shape)
