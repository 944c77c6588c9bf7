"""Write-back helper (``src/squidpy/gr/_utils.py:77-86``) and small host utilities."""

from __future__ import annotations

import logging
import time
from typing import Any, NamedTuple

import numpy as np

from .._device import DevSparse, array_device, device_graph, graph_args
from .._lib import pointer_device

logg = logging.getLogger("squidpy_b200")


def _save_data(adata: Any, *, attr: str, key: str, data: Any, prefix: bool = True, time_start: float | None = None) -> None:
    obj = getattr(adata, attr)
    obj[key] = data
    logg.info("Adding `adata.%s[%r]`", attr, key) if prefix else logg.info("       `adata.%s[%r]`", attr, key)
    if time_start is not None:
        logg.info("Finish (%.3fs)", time.perf_counter() - time_start)


def category_codes(series, *, dtype) -> tuple[np.ndarray, int]:
    """Category -> code mapping of the reference (``clust_map`` dict loop, ``gr/_nhood.py:194-197``): code = position in
    ``cat.categories``.  A missing value has no entry in that dict and raises ``KeyError`` there; same here."""
    # the Categorical's own code array: `series.cat.codes` would build a Series carrying the (string) obs index first
    codes = np.asarray(series.array.codes if hasattr(series, "array") else series.cat.codes)
    if (codes < 0).any():
        raise KeyError(float("nan"))
    return codes.astype(dtype), len(series.cat.categories)


def var_positions(var_names, genes) -> np.ndarray:
    """``adata[:, genes]`` as int64 column positions: ``genes`` holds var names, or integer positions."""
    import pandas as pd

    sel = np.asarray(genes)
    if sel.dtype.kind in "iu":
        return sel.astype(np.int64)
    ix = pd.Index(var_names).get_indexer(sel)
    if (ix < 0).any():
        raise KeyError(f"Values {[str(s) for s, i in zip(sel, ix) if i < 0]} are not valid var names or indices.")
    return ix.astype(np.int64)


def as_csr(mat):
    import scipy.sparse as sp

    if sp.issparse(mat) and mat.format == "csr":
        return mat
    return sp.csr_matrix(mat)


def graph_device(d: DevSparse, device: int | None) -> int:
    """The CUDA device holding a device graph; an explicit ``device`` must name it."""
    on = array_device(d, pointer_device)
    if device is not None and int(device) != on:
        raise ValueError(f"`device={device}` does not match the device of the connectivity graph, cuda:{on}.")
    return on


class CallerGraph(NamedTuple):
    """An ``n x n`` neighbour graph for the C entry points that rebuild it (``sqb_centrality_scores``, ``sqb_niche_*``).

    ``index_args`` are its ``(n, nnz, indptr, indptr_bits, indices, index_bits)`` arguments: the pointers of its CSR arrays (a
    CSC's are the CSR of its transpose), int32 / int64.  The values are left to the caller: ``host`` is the scipy CSR / CSC of a
    host graph, ``dev`` the description of a device graph (the other one is ``None``)."""

    index_args: tuple
    csc: bool
    host: Any
    dev: DevSparse | None
    device: int | None  # the device holding a device graph, else the one asked for
    stream: int  # a device graph's producer stream, 0 for a host graph
    keep: tuple  # the host index arrays behind index_args


def caller_graph(conn: Any, n: int, device: int | None) -> CallerGraph:
    """``conn`` (scipy / numpy on the host, or a CSR / CSC in GPU memory) checked to be ``n x n`` and described for the C ABI."""
    import scipy.sparse as sp

    dev = device_graph(conn)
    if dev is None:
        g = conn if sp.issparse(conn) and conn.format in ("csr", "csc") else as_csr(conn)
        if g.shape != (n, n):
            raise ValueError(f"Expected the connectivity graph to be of shape `{(n, n)}`, found `{g.shape}`.")
        indptr, indices = (np.ascontiguousarray(a) if a.dtype in (np.int32, np.int64) else np.ascontiguousarray(a, np.int64)
                           for a in (g.indptr, g.indices))
        return CallerGraph((n, indices.size, indptr.ctypes.data, 8 * indptr.itemsize, indices.ctypes.data, 8 * indices.itemsize),
                           g.format == "csc", g, None, device, 0, (indptr, indices))
    graph = graph_args(dev, n)
    return CallerGraph((n, graph.nnz, graph.indptr, graph.indptr_bits, graph.indices or None, graph.index_bits), graph.transposed, None,
                       dev, graph_device(dev, device), graph.stream, ())
