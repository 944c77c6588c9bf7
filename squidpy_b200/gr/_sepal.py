"""``sepal`` — drop-in for ``squidpy.gr.sepal`` (``src/squidpy/gr/_sepal.py:31-183``): spatially variable genes by simulated
diffusion on the spot lattice, with the per-gene diffusion loop (up to ``n_iter`` dependent iterations) on the H100
(``sqb_sepal``: one CTA per gene, the field in shared memory).  The one-off neighbourhood bookkeeping (`_compute_idxs`:
saturated / unsaturated nodes, nearest saturated node of the border spots) stays on the host."""

from __future__ import annotations

import time
from collections.abc import Sequence
from typing import Any

import numpy as np
import pandas as pd
from scipy.sparse import csr_matrix, issparse

from .._constants import Key
from .._device import DevMatrix, device_matrix, on_host
from .._lib import Context, check, default_context, load
from .._validators import assert_connectivity_key, assert_spatial_basis, extract_adata_if_sdata
from ._gather import GENE_MAJOR, Gathered, device_context
from ._utils import _save_data, logg, var_positions

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
    and ignored."""
    adata = extract_adata_if_sdata(adata, table_key=table_key)
    assert_connectivity_key(adata, connectivity_key)
    assert_spatial_basis(adata, key=spatial_key)
    if max_neighs not in (4, 6):
        raise ValueError(f"Expected `max_neighs` to be either `4` or `6`, found `{max_neighs}`.")
    spatial = np.asarray(on_host(adata.obsm[spatial_key])).astype(np.float64)
    if genes is None:
        genes = adata.var_names.values
        if "highly_variable" in adata.var.columns:
            genes = genes[adata.var["highly_variable"].values]
    genes = [genes] if isinstance(genes, str) else list(dict.fromkeys(genes))
    if not genes:
        raise ValueError("No genes have been selected.")

    g = on_host(adata.obsp[connectivity_key])
    g = g.copy() if (issparse(g) and g.format == "csr") else csr_matrix(g)
    g.eliminate_zeros()
    max_n = np.diff(g.indptr).max()
    if max_n != max_neighs:
        raise ValueError(f"Expected `max_neighs={max_neighs}`, found node with `{max_n}` neighbors.")
    sat, sat_idx, unsat, unsat_idx = _compute_idxs(g, spatial, max_neighs)

    if use_raw and adata.raw is None:
        use_raw = False
    src = adata.raw if use_raw else adata
    if use_raw:
        genes = list(set(src.var_names) & set(genes))
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
        logg.info("Calculating sepal score for `%d` genes on the GPU", len(genes))
        score = _scores_device(m, ctx, positions, sat, sat_idx, unsat, unsat_idx, max_neighs=max_neighs, n_iter=int(n_iter),
                               dt=dt, thresh=thresh, batch_genes=None)
    else:
        sub = src[:, genes]
        vals = sub.X if (layer is None or use_raw) else sub.layers[layer]
        start = time.perf_counter()
        logg.info("Calculating sepal score for `%d` genes on the GPU", len(genes))
        score = sepal_scores(vals, sat, sat_idx, unsat, unsat_idx, max_neighs=max_neighs, n_iter=int(n_iter), dt=dt, thresh=thresh,
                             ctx=default_context(device))
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
