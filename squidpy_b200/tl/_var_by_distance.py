"""``var_by_distance`` — drop-in for ``squidpy.tl.var_by_distance`` (``src/squidpy/tl/_var_by_distance.py:22-258``).

The expensive step of the reference is ``KDTree(anchor_coord).query(batch_coord)`` for every (slide, anchor) combination
(:129-134), followed by pandas work keyed on obs names: a boolean ``adata[mask]`` per combination, merges and reindexing.
Here every combination's search runs in ONE call of the exact nearest-anchor kernel (``sqb_nn_min_dist_f64``: float64
distances bit-identical to scikit-learn's KDTree for its three metric classes), on one pool of points: per slide, its
observations with finite coordinates (the query range shared by that slide's anchors), followed by the anchor sets.  The
frame is then built by position: per-slide normalisation on arrays and one DataFrame construction, with the reference's
column order, dtypes, row order and NaN placement.
"""

from __future__ import annotations

import time
from typing import Any

import numpy as np
import pandas as pd

from .._device import on_host
from .._lib import Context, check, default_context, load
from .._metrics import metric_code
from ..gr._utils import _save_data, logg

__all__ = ["var_by_distance", "nn_min_dist", "metric_code"]


def nn_min_dist(points: np.ndarray, tasks: np.ndarray, metric: int, n_out: int, *, ctx: Context | None = None) -> np.ndarray:
    """Distance from every query point to its nearest reference point, on the GPU: float64 (n_out,).

    ``points`` is an (n, 2) pool of finite float64 coordinates; every row of ``tasks`` (int64, 5 columns) is ``(ref_begin,
    ref_end, qry_begin, qry_end, out_begin)``: ``out[out_begin + (q - qry_begin)]`` is the distance from ``points[q]`` to its
    nearest point of ``points[ref_begin:ref_end]`` (non-empty; no point excluded), i.e.
    ``KDTree(ref, metric=DistanceMetric.get_metric(m)).query(qry)[0]`` bit for bit.  ``metric``: see :func:`metric_code`.
    Output ranges must not overlap; positions no task writes are NaN."""
    lib = load()
    ctx = ctx or default_context()
    pts = np.ascontiguousarray(np.asarray(points, dtype=np.float64).reshape(-1, 2))
    tk = np.ascontiguousarray(np.asarray(tasks, dtype=np.int64).reshape(-1, 5))
    out = np.empty(int(n_out), dtype=np.float64)
    check(lib.sqb_nn_min_dist_f64(ctx.handle, pts.ctypes.data, pts.shape[0], tk.ctypes.data, tk.shape[0], int(metric), out.size, out.ctypes.data))
    return out


def _take(series: pd.Series, pos: np.ndarray) -> Any:
    """``series`` at positions ``pos`` (-1: missing, filled the way ``reindex`` fills: NaN, with its dtype promotion)."""
    values = series.array
    if isinstance(series.dtype, np.dtype):
        return pd.api.extensions.take(np.asarray(values), pos, allow_fill=True)
    return values.take(pos, allow_fill=True)


def var_by_distance(
    adata: Any,
    groups: str | list[str] | np.ndarray,
    cluster_key: str | None = None,
    library_key: str | None = None,
    library_id: str | list[str] | None = None,
    design_matrix_key: str = "design_matrix",
    covariates: str | list[str] | None = None,
    metric: str = "euclidean",
    spatial_key: str = "spatial",
    copy: bool = False,
    *,
    device: int | None = None,
) -> pd.DataFrame | None:
    """Build a design matrix of distances from every observation to the nearest observation of each anchor.

    Parameters as ``squidpy.tl.var_by_distance``: ``groups`` names anchor clusters of ``adata.obs[cluster_key]`` (a str, a
    list, or a 1-D ndarray of names), or is a list of coordinate pairs (one custom anchor per slide).  Distances are computed
    per slide of ``adata.obs[library_key]`` (restricted to ``library_id``) with ``metric`` (any ``KDTree`` metric name),
    from the coordinates of ``adata.obsm["spatial"]``; rows with a NaN coordinate in ``adata.obsm[spatial_key]`` get NaN.
    Each anchor ``a`` gives the columns ``a`` (normalised per slide: zeros become NaN, the first minimum 0, divided by the
    slide's maximum) and ``a_raw``.  ``covariates`` are copied from ``adata.obs``.  ``device``: the CUDA device (default:
    the context of ``squidpy_b200.default_context``).

    Coordinates must be 2-D: other shapes raise ``NotImplementedError``.

    Returns the design matrix if ``copy=True``, else stores it in ``adata.obsm[design_matrix_key]``."""
    start = time.perf_counter()
    logg.info("Creating %s", design_matrix_key)

    if isinstance(groups, str):
        anchor: list = [groups]
    elif isinstance(groups, list):
        anchor = groups
    elif isinstance(groups, np.ndarray):
        if groups.ndim != 1:
            raise ValueError(f"Expected a 1D array for 'groups', but got shape {groups.shape}.")
        anchor = groups.astype(str).tolist()
    else:
        raise TypeError(f"Expected `groups` to be of type `str or list or ndarray`, got `{type(groups).__name__}`.")

    obs = adata.obs
    batch: list
    if library_key is None:
        batch = [None]
    elif isinstance(library_key, str):
        slides = obs[library_key].unique()
        if library_id is not None:
            if isinstance(library_id, str):
                library_id = [library_id]
            for x in library_id:
                if x not in slides:
                    raise ValueError(f"library id {x} not in {library_key}")
            batch = [s for s in library_id if s in slides]
        else:
            batch = slides.tolist()
    else:
        raise TypeError(f"Expected `library_key` to be of type `str`, got `{type(library_key).__name__}`.")

    if all(isinstance(x, list) for x in anchor):
        if len(anchor) != len(batch):
            raise ValueError(f"There must be one anchor point per slide. A numpy array with {len(anchor)} anchor points was provided, "
                             f"but {len(batch)} slides were found.")
        combinations = list(zip(anchor, batch))
    else:
        combinations = [(a, b) for a in anchor for b in batch]

    coords = np.asarray(on_host(adata.obsm["spatial"]), dtype=np.float64)
    if coords.ndim != 2 or coords.shape[1] != 2:
        raise NotImplementedError(f"var_by_distance on the GPU takes 2-D coordinates, found `adata.obsm['spatial']` of shape {coords.shape}.")
    n = coords.shape[0]
    finite = ~np.isnan(coords).any(axis=1)
    nan_src = coords if spatial_key == "spatial" else np.asarray(on_host(adata.obsm[spatial_key]))
    nan_row = np.isnan(nan_src).reshape(nan_src.shape[0], -1).any(axis=1)
    cl = obs[cluster_key] if cluster_key is not None else None
    with_cluster = library_key is not None and cluster_key is not None
    base = ([cluster_key, library_key] if with_cluster else [library_key]) if library_key is not None else \
        ([cluster_key] if cluster_key is not None else [])
    anchor_col = 2 if with_cluster else 1

    # one pool for every combination: per slide its finite rows (the shared query range), then each anchor set
    slide_rows: dict = {}
    blocks: list[np.ndarray] = []
    tasks: list[tuple[int, int, int, int, int]] = []
    combos: dict = {}  # (slide, anchor name) -> (rows, out_begin); insertion order is the reference's
    code = None
    pool_n = out_n = 0
    anchor_mask: dict = {}
    for anchor_var, batch_var in combinations:
        if batch_var not in slide_rows:
            rows = np.arange(n) if batch_var is None else np.flatnonzero(np.asarray(obs[library_key] == batch_var, dtype=bool))
            q = rows[finite[rows]]
            slide_rows[batch_var] = (rows, q, pool_n)
            blocks.append(coords[q])
            pool_n += q.size
        rows, q, q0 = slide_rows[batch_var]
        if with_cluster and anchor_var not in pd.unique(cl.iloc[rows]):
            continue
        if code is None:
            code = metric_code(metric)
        if isinstance(anchor_var, list):
            pts = np.array(anchor_var).reshape(1, -1)
            if pts.shape[1] != 2:
                raise ValueError(f"query data dimension must match training data dimension: anchor {anchor_var} for 2-D coordinates")
            pts = pts.astype(np.float64)
        else:
            if anchor_var not in anchor_mask:
                anchor_mask[anchor_var] = np.asarray(obs[cluster_key] == anchor_var, dtype=bool)
            sel = q[anchor_mask[anchor_var][q]]
            pts = coords[sel]
        if pts.shape[0] == 0:
            raise ValueError(f"Found array with 0 sample(s) (shape=(0, 2)) while a minimum of 1 is required by KDTree: no anchor `{anchor_var}`.")
        if isinstance(anchor_var, list) and all(isinstance(x, (int, float)) for x in anchor_var):
            anchor_var = "custom_anchor"
            anchor = ["custom_anchor"]
        if anchor_col > len(base):
            raise IndexError(f"index {anchor_col} is out of bounds for the design matrix's {len(base)} columns")
        blocks.append(pts)
        tasks.append((pool_n, pool_n + pts.shape[0], q0, q0 + q.size, out_n))
        combos[(batch_var, str(anchor_var))] = (rows, q, out_n)
        pool_n += pts.shape[0]
        out_n += q.size

    pool = np.concatenate(blocks) if blocks else np.zeros((0, 2))
    dist = nn_min_dist(pool, np.asarray(tasks, dtype=np.int64).reshape(-1, 5), code, out_n, ctx=default_context(device)) if tasks else np.zeros(0)

    # per combination: NaN rows re-inserted (at the NaN rows of obsm[spatial_key]), raw and normalised distances
    norm: dict = {}
    for key, (rows, q, o) in combos.items():
        nan_ids = np.flatnonzero(nan_row[rows])
        d = np.insert(dist[o : o + q.size], nan_ids - np.arange(nan_ids.size), np.nan)
        if d.size != rows.size:
            raise ValueError(f"Length of values ({d.size}) does not match length of index ({rows.size})")
        v = np.where(d == 0, np.nan, d)
        v[np.nanargmin(v)] = 0.0
        with np.errstate(invalid="ignore", divide="ignore"):
            v = v / np.nanmax(v)
        norm[key] = (rows, v, d)

    def columns_of(name: str) -> list:
        return base[:anchor_col] + [name] + base[anchor_col:] + [f"{name}_raw"]

    index_name = obs.index.name
    cols: dict = {}
    if library_key is None:
        order = np.arange(n)
        if len(anchor) > 1:  # inner merges on (cluster, obs), then obs as the index
            if cluster_key is None:
                raise KeyError(None)
            names = columns_of(str(anchor[0]))
            for (_, a) in list(norm)[1:]:
                names += [a, f"{a}_raw"]
            if not isinstance(groups, list):
                index_name = None
        else:
            names = columns_of(str(anchor[0]))
        for (_, a), (rows, v, d) in norm.items():
            cols[a], cols[f"{a}_raw"] = v, d
        for c in base:
            cols[c] = _take(obs[c], order)
    else:
        per_anchor = list(dict.fromkeys(str(x) for x in anchor))
        names = columns_of(per_anchor[0])
        for a in per_anchor[1:]:  # the outer merges add each frame's new columns, sorted (Index.difference)
            names += sorted(set(columns_of(a)) - set(names))
        order = np.arange(n) if len(anchor) == 1 or isinstance(groups, list) else np.asarray(obs.index.argsort())
        for i, a in enumerate(per_anchor):
            src = [(rows, v, d) for (_, b), (rows, v, d) in norm.items() if b == a]
            if not src:
                raise ValueError("No objects to concatenate")
            pos = np.full(n, -1, dtype=np.int64)
            val, raw = np.full(n, np.nan), np.full(n, np.nan)
            for rows, v, d in src:
                pos[rows], val[rows], raw[rows] = rows, v, d
            cols[a], cols[f"{a}_raw"] = val[order], raw[order]
            if i == 0:
                for c in base:
                    cols[c] = _take(obs[c], pos[order])
    index = obs.index.take(order)
    df = pd.DataFrame({name: cols[name] for name in names}, index=index)
    df.index.name = index_name

    if covariates is not None:
        if isinstance(covariates, str):
            covariates = [covariates]
        for c in covariates:
            df[c] = _take(obs[c], order)
    if copy:
        logg.info("Finish (%.3fs)", time.perf_counter() - start)
        return df
    _save_data(adata, attr="obsm", key=design_matrix_key, data=df, time_start=start)
    return None
