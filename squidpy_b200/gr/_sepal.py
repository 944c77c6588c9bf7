"""``sepal`` — drop-in for ``squidpy.gr.sepal`` (``src/squidpy/gr/_sepal.py:31-183``): spatially variable genes by simulated
diffusion on the spot lattice, with the per-gene diffusion loop (up to ``n_iter`` dependent iterations) on the H100
(``sqb_sepal``: one CTA per gene, the field in shared memory).  The one-off neighbourhood bookkeeping (`_compute_idxs`:
saturated / unsaturated nodes, nearest saturated node of the border spots) is built on the GPU too (``sqb_sepal_idxs``), from
a CSR / CSC graph on the host or read in place in GPU memory (``sepal_idxs``)."""

from __future__ import annotations

import ctypes as C
import time
from collections.abc import Sequence
from typing import Any

import numpy as np
import pandas as pd
from scipy.sparse import csr_matrix, issparse

from .._constants import Key
from .._device import DevArray, DevMatrix, DevSparse, _contiguous_1d, device_matrix, on_host
from .._dist import all_gather_rows, broadcast_from_rank0, shard_range, world
from .._lib import Context, check, default_context, load, pointer_device
from .._validators import assert_connectivity_key, assert_spatial_basis, extract_adata_if_sdata
from ._gather import GENE_MAJOR, Gathered, device_context
from ._utils import _save_data, caller_graph, logg, var_positions

__all__ = ["sepal", "sepal_scores"]


def _compute_idxs(g: csr_matrix, spatial: np.ndarray, sat_thresh: int):
    """``_compute_idxs`` (``_sepal.py:292-358``): nodes with exactly ``sat_thresh`` neighbours are saturated; every other node
    follows its first saturated neighbour (CSR order) or, without one, the saturated node nearest in L1 distance."""
    from sklearn.metrics import pairwise_distances

    n_indices = np.diff(g.indptr)
    unsat = np.flatnonzero(n_indices < sat_thresh)
    sat = np.flatnonzero(n_indices == sat_thresh)
    starts = g.indptr[sat]
    sat_idx = g.indices[starts[:, None] + np.arange(sat_thresh)[None, :]].astype(np.int32)
    is_sat = np.zeros(g.shape[0], dtype=bool)
    is_sat[sat] = True
    nearest = np.full(unsat.shape[0], np.nan)
    for k, i in enumerate(unsat):
        nb = g.indices[g.indptr[i] : g.indptr[i + 1]]
        hit = nb[is_sat[nb]]
        if hit.size:
            nearest[k] = hit[0]
    missing = np.isnan(nearest)
    if missing.any():
        dist = pairwise_distances(spatial[unsat[missing]], spatial[sat], metric="l1")
        nearest[missing] = sat[np.argmin(dist, axis=1)]
    return sat.astype(np.int32), sat_idx, unsat.astype(np.int32), nearest.astype(np.int32)


# value dtype codes of sqb_sepal_idxs; a host graph of another dtype passes `data != 0`, the only thing the tables read
_VALUE_CODES = {np.dtype(np.float32): 0, np.dtype(np.float64): 1, np.dtype(np.int32): 3, np.dtype(np.int64): 4, np.dtype(np.bool_): 5}


def _device_graph_ok(d: DevSparse, n: int) -> bool:
    """Whether sqb_sepal_idxs reads the device graph ``d`` in place: an ``n x n`` CSR / CSC on one device, with contiguous int32 /
    int64 index arrays, ``nnz < 2^31`` contiguous values of a dtype in ``_VALUE_CODES`` and at most one producer stream."""
    ints = (np.dtype(np.int32), np.dtype(np.int64))
    if tuple(d.shape) != (n, n) or d.indptr.dtype not in ints or d.indices.dtype not in ints or d.data.dtype not in _VALUE_CODES:
        return False
    nnz = d.indices.shape[0] if len(d.indices.shape) == 1 else -1
    if not (_contiguous_1d(d.indptr, n + 1) and _contiguous_1d(d.indices) and _contiguous_1d(d.data, nnz)) or nnz >= 1 << 31:
        return False
    devices = {pointer_device(a.ptr) for a in d.arrays if a.ptr}
    return len(devices) == 1 and min(devices) >= 0 and len({a.stream for a in d.arrays if a.stream}) <= 1


def _graph_abi(conn: Any, n: int, device: int | None) -> tuple[tuple, Any, int | None] | None:
    """``(graph arguments of sqb_sepal_idxs, owner, device)`` of a host graph (run on ``device``) or of a CSR / CSC in GPU memory
    (run on the graph's device), or ``None`` for a graph the tables are built from on the host (dense device graphs, float16 and
    other device dtypes, graphs that are not square)."""
    dev = device_matrix(conn)
    if n < 1 or tuple(conn.shape) != (n, n) or (dev is not None and not (isinstance(dev, DevSparse) and _device_graph_ok(dev, n))):
        return None
    if dev is None:
        host = conn if issparse(conn) and conn.format in ("csr", "csc") else csr_matrix(conn)
        if host.nnz >= 1 << 31:
            return None
        g = caller_graph(host, n, device)
        code = _VALUE_CODES.get(host.data.dtype)
        data = np.ascontiguousarray(host.data) if code is not None else np.ascontiguousarray(host.data != 0)
        code, ptr = 5 if code is None else code, data.ctypes.data
    else:
        g = caller_graph(conn, n, None)  # on the graph's own device, whatever `device` names
        data, code, ptr = dev.data, _VALUE_CODES[dev.data.dtype], dev.data.ptr or None
    return (*g.index_args, ptr, code, int(g.csc), int(g.dev is not None), g.stream), (g, data), g.device


def _xy_abi(spatial: Any, n: int, device: int) -> tuple[tuple, Any] | None:
    """``(coordinate arguments of sqb_sepal_idxs, owner)``: an ``n x 2`` float32 / float64 device array on ``device`` in place,
    anything else as the host path converts it (float64), or ``None`` when that is not ``n x 2``."""
    d = device_matrix(spatial)
    if (isinstance(d, DevArray) and tuple(d.shape) == (n, 2) and d.dtype in (np.dtype(np.float32), np.dtype(np.float64))
            and pointer_device(d.ptr) == device):
        return (d.ptr, int(d.dtype == np.float64), d.strides[0], d.strides[1], 1, d.stream), d
    xy = np.ascontiguousarray(np.asarray(on_host(spatial)).astype(np.float64, copy=False))
    if xy.shape != (n, 2):
        return None
    return (xy.ctypes.data, 1, 2, 1, 0, 0), xy


def _host_idxs(conn: Any, spatial: Any, max_neighs: int):
    """The tables from host copies of the graph and the coordinates, through ``_compute_idxs``."""
    g = on_host(conn)
    g = g.copy() if (issparse(g) and g.format == "csr") else csr_matrix(g)
    g.eliminate_zeros()
    max_n = np.diff(g.indptr).max()
    if max_n != max_neighs:
        raise ValueError(f"Expected `max_neighs={max_neighs}`, found node with `{max_n}` neighbors.")
    return _compute_idxs(g, np.asarray(on_host(spatial)).astype(np.float64), max_neighs)


def sepal_idxs(conn: Any, spatial: Any, max_neighs: int, *, device: int | None = None):
    """``(sat, sat_idx, unsat, unsat_idx)`` of ``_compute_idxs`` for the graph ``conn`` after ``eliminate_zeros``, with the
    reference's ``max_neighs`` check first, built on the GPU (``sqb_sepal_idxs``).

    A host graph (converted to CSR unless it is a CSR / CSC) is built from on ``device``; a CSR / CSC in GPU memory (cupyx-style
    or torch ``sparse_csr`` / ``sparse_csc``) is read in place on its own device.  ``spatial`` (``n x 2``) is read in place when
    it is a float32 / float64 array on that device, else converted to float64 on the host.  Other inputs (dense device graphs,
    float16 device values, coordinates that are not ``n x 2``) take ``_compute_idxs`` on host copies, as do non-finite
    coordinates of an orphan or a saturated node, which scikit-learn's ``pairwise_distances`` refuses there."""
    n = conn.shape[0]
    graph = _graph_abi(conn, n, device)
    ctx = None if graph is None else default_context(graph[2])
    xy = None if ctx is None else _xy_abi(spatial, n, ctx.device)
    if xy is None:
        return _host_idxs(conn, spatial, max_neighs)
    (g_args, g_keep, _), (xy_args, xy_keep) = graph, xy
    k = int(max_neighs)
    sat, sat_idx, unsat, unsat_idx = (np.empty(m, dtype=np.int32) for m in (n, n * max(k, 0), n, n))
    max_deg, n_sat, n_unsat, bad = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int()
    with ctx.lock:
        check(load().sqb_sepal_idxs(ctx.handle, *g_args, *xy_args, k, C.byref(max_deg), sat.ctypes.data, sat_idx.ctypes.data, unsat.ctypes.data,
                                    unsat_idx.ctypes.data, C.byref(n_sat), C.byref(n_unsat), C.byref(bad)))
    del g_keep, xy_keep
    if max_deg.value != max_neighs:
        raise ValueError(f"Expected `max_neighs={max_neighs}`, found node with `{max_deg.value}` neighbors.")
    if bad.value:
        return _host_idxs(conn, spatial, max_neighs)  # raises scikit-learn's error, as the host path does
    ns, nu = n_sat.value, n_unsat.value
    return sat[:ns], sat_idx[: ns * k].reshape(ns, k), unsat[:nu], unsat_idx[:nu]


def sepal_scores(vals: Any, sat, sat_idx, unsat, unsat_idx, *, max_neighs: int, n_iter: int = 30000, dt: float = 0.001,
                 thresh: float = 1e-8, ctx: Context | None = None, batch_genes: int | None = None) -> np.ndarray:
    """``_diffusion_genes`` (``_sepal.py:186-233``): ``vals`` observations x genes (dense or scipy sparse, or a matrix in GPU
    memory: see ``sepal``) -> float64 score per gene.  The genes are scored in batches of ``batch_genes`` (default: as many as
    fill 1 GB of dense float64)."""
    if device_matrix(vals) is not None:
        m, on = device_context(vals, None if ctx is None else ctx.device)
        return _scores_device(m, ctx or on, np.arange(m.shape[1]), sat, sat_idx, unsat, unsat_idx, max_neighs=max_neighs, n_iter=n_iter, dt=dt,
                              thresh=thresh, batch_genes=batch_genes)
    lib = load()
    ctx = ctx or default_context()
    n, n_genes = vals.shape
    out = np.empty(n_genes, dtype=np.float64)
    sat = np.ascontiguousarray(sat, dtype=np.int32)
    sat_idx = np.ascontiguousarray(sat_idx, dtype=np.int32)
    unsat = np.ascontiguousarray(unsat, dtype=np.int32)
    unsat_idx = np.ascontiguousarray(unsat_idx, dtype=np.int32)
    step = _batch(n, n_genes, batch_genes)
    sparse = issparse(vals)
    if sparse:
        vals = vals.tocsc()
    with ctx.lock:
        for g0 in range(0, n_genes, step):
            g1 = min(g0 + step, n_genes)
            blk = vals[:, g0:g1]
            dense = np.ascontiguousarray((blk.toarray() if sparse else np.asarray(blk)).T, dtype=np.float64)  # genes x observations
            check(lib.sqb_sepal(ctx.handle, dense.ctypes.data, g1 - g0, n, sat.ctypes.data, sat.size, sat_idx.ctypes.data, int(max_neighs),
                                unsat.ctypes.data, unsat_idx.ctypes.data, unsat.size, int(n_iter), float(dt), float(thresh), out[g0:g1].ctypes.data))
    return out


def _batch(n: int, n_genes: int, batch_genes: int | None) -> int:
    if batch_genes is not None:
        if int(batch_genes) < 1:
            raise ValueError(f"Expected `batch_genes` to be positive, found `{batch_genes}`.")
        return min(n_genes, int(batch_genes))
    return max(1, min(n_genes, (1 << 30) // (8 * max(n, 1))))  # <= 1 GB of dense float64 per device call


def _scores_device(m: DevMatrix, ctx: Context, positions: np.ndarray, sat, sat_idx, unsat, unsat_idx, *, max_neighs: int, n_iter: int,
                   dt: float, thresh: float, batch_genes: int | None) -> np.ndarray:
    """``sepal_scores`` of the columns ``positions`` of a device matrix: every batch is gathered on the device (genes x
    observations, float64, NaN kept as the host path keeps it) and scored there."""
    lib = load()
    n, n_genes = m.shape[0], len(positions)
    out = np.empty(n_genes, dtype=np.float64)
    sat = np.ascontiguousarray(sat, dtype=np.int32)
    sat_idx = np.ascontiguousarray(sat_idx, dtype=np.int32)
    unsat = np.ascontiguousarray(unsat, dtype=np.int32)
    unsat_idx = np.ascontiguousarray(unsat_idx, dtype=np.int32)
    step = _batch(n, n_genes, batch_genes)
    with ctx.lock:
        for g0 in range(0, n_genes, step):
            g1 = min(g0 + step, n_genes)
            with Gathered(ctx, m, None, positions[g0:g1], GENE_MAJOR, nan_zero=False) as x:
                check(lib.sqb_sepal_dense(x.handle, sat.ctypes.data, sat.size, sat_idx.ctypes.data, int(max_neighs), unsat.ctypes.data,
                                          unsat_idx.ctypes.data, unsat.size, int(n_iter), float(dt), float(thresh), out[g0:g1].ctypes.data))
    return out


def sepal(adata: Any, max_neighs: int, genes: str | Sequence[str] | None = None, n_iter: int | None = 30000, dt: float = 0.001,
          thresh: float = 1e-8, connectivity_key: str = Key.obsp.spatial_conn(), spatial_key: str = Key.obsm.spatial, layer: str | None = None,
          use_raw: bool = False, copy: bool = False, n_jobs: int | None = None, show_progress_bar: bool = True, *, table_key: str | None = None,
          device: int | None = None) -> pd.DataFrame | None:
    """Identify spatially variable genes with *Sepal* (see module docstring).  Returns / writes ``adata.uns['sepal_score']``: a
    DataFrame indexed by gene with the column ``sepal_score``, sorted descending.  ``n_jobs`` / ``show_progress_bar`` are accepted
    and ignored.
    Under an initialised ``torch.distributed`` process group (one process per GPU) the genes are sharded over the ranks and the
    scores all-gathered once; every rank gets the full result."""
    adata = extract_adata_if_sdata(adata, table_key=table_key)
    assert_connectivity_key(adata, connectivity_key)
    assert_spatial_basis(adata, key=spatial_key)
    if max_neighs not in (4, 6):
        raise ValueError(f"Expected `max_neighs` to be either `4` or `6`, found `{max_neighs}`.")
    spatial = adata.obsm[spatial_key]
    if device_matrix(spatial) is None:  # device coordinates are read where they live (sepal_idxs)
        spatial = np.asarray(spatial).astype(np.float64)
    if genes is None:
        genes = adata.var_names.values
        if "highly_variable" in adata.var.columns:
            genes = genes[adata.var["highly_variable"].values]
    genes = [genes] if isinstance(genes, str) else list(dict.fromkeys(genes))
    if not genes:
        raise ValueError("No genes have been selected.")

    sat, sat_idx, unsat, unsat_idx = sepal_idxs(adata.obsp[connectivity_key], spatial, max_neighs, device=device)

    if use_raw and adata.raw is None:
        use_raw = False
    src = adata.raw if use_raw else adata
    if use_raw:
        # set order follows the process's string hashing, which differs between ranks: every rank takes rank 0's order, so
        # that a gene's position, and with it its shard, means the same gene everywhere
        genes = broadcast_from_rank0(list(set(src.var_names) & set(genes)))
    rank, ws = world()
    lo, hi = shard_range(len(genes), rank, ws)
    whole = src.X if (layer is None or use_raw) else src.layers[layer]
    if device_matrix(whole) is not None:  # the genes are gathered by position on the array's device; X is not read on the host
        m, ctx = device_context(whole, device)
        if m.shape[0] != adata.shape[0]:
            raise ValueError(f"Expected the expression matrix to have `{adata.shape[0]}` rows, found `{m.shape[0]}`.")
        positions = var_positions(src.var_names, genes)  # names or integer positions, as src[:, genes] takes them
        if ((positions < -m.shape[1]) | (positions >= m.shape[1])).any():
            raise IndexError(f"Gene positions must lie in [-{m.shape[1]}, {m.shape[1]}).")
        positions = positions % m.shape[1]  # negative positions count from the end, as in X[:, genes]
        start = time.perf_counter()
        logg.info("Calculating sepal score for `%d` genes on cuda:%d (rank %d/%d, genes %d..%d)", len(genes), ctx.device, rank, ws, lo, hi)
        score = _scores_device(m, ctx, positions[lo:hi], sat, sat_idx, unsat, unsat_idx, max_neighs=max_neighs, n_iter=int(n_iter),
                               dt=dt, thresh=thresh, batch_genes=None)
    else:
        sub = src[:, genes]
        vals = sub.X if (layer is None or use_raw) else sub.layers[layer]
        if ws > 1:
            vals = vals[:, lo:hi]
        ctx = default_context(device)
        start = time.perf_counter()
        logg.info("Calculating sepal score for `%d` genes on cuda:%d (rank %d/%d, genes %d..%d)", len(genes), ctx.device, rank, ws, lo, hi)
        score = sepal_scores(vals, sat, sat_idx, unsat, unsat_idx, max_neighs=max_neighs, n_iter=int(n_iter), dt=dt, thresh=thresh, ctx=ctx)
    score = all_gather_rows(score, len(genes))
    key_added = "sepal_score"
    sepal_score = pd.DataFrame(score, index=genes, columns=[key_added])
    if sepal_score[key_added].isna().any():
        logg.warning("Found `NaN` in sepal scores, consider increasing `n_iter` to a higher value")
    sepal_score = sepal_score.sort_values(by=key_added, ascending=False)
    if copy:
        logg.info("Finish (%.3fs)", time.perf_counter() - start)
        return sepal_score
    _save_data(adata, attr="uns", key=key_added, data=sepal_score, time_start=start)
    return None
