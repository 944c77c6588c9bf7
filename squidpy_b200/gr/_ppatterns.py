"""``spatial_autocorr`` and ``co_occurrence`` — drop-ins for ``squidpy.gr.spatial_autocorr`` / ``co_occurrence``
(``src/squidpy/gr/_ppatterns.py:56-255`` and ``:361-428``) with the hot loops on an H100.

* Moran's I / Geary's C for every feature: CUDA (``sqb_autocorr_*``) instead of ``scanpy.metrics.morans_i/gearys_c``
  (``_ppatterns.py:216,267-272``).  ``adata.X`` in its native CSR (cells x genes) layout is consumed directly — the
  reference's ``.T`` + CSC->CSR conversion happens on the device.
* Co-occurrence pair counting: CUDA (``sqb_cooc_counts``) instead of ``_occur_count`` (``_ppatterns.py:283-310``).
* Analytic moments / p-values, FDR correction, probability normalisation stay on the host and follow the reference's
  formulas and dtypes (float32 moments, ``_ppatterns.py:443-559``; occ ratio ``:347-356``).
"""

from __future__ import annotations

import ctypes as C
import time
import warnings
from collections.abc import Sequence
from typing import Any, Literal, NamedTuple

import numpy as np
import pandas as pd
from scipy import stats
from scipy.sparse import issparse, spmatrix

from .._constants import Key, SpatialAutocorr
from .._device import (DevArray, DevGraph, DevSparse, array_device, common_stream, device_matrix, dtype_code, feature_map, index_bits,
                       on_host, to_host_matrix, weight_graph_args)
from .._dist import all_gather_rows, all_reduce_sum, shard_range, shared_seed, world
from .._lib import Context, check, default_context, load, pointer_device
from .._rng import spawn_generators
from .._validators import (
    assert_categorical_obs,
    assert_connectivity_key,
    assert_key_in_adata,
    assert_positive,
    assert_spatial_basis,
    extract_adata_if_sdata,
)
from ._utils import _save_data, as_csr, category_codes, logg, var_positions

__all__ = ["spatial_autocorr", "co_occurrence", "AutocorrPlan", "cooc_counts"]

fp = np.float32
ip = np.int32
SQB_ERR_LAYOUT = -6  # sqb_autocorr_create_device: a row of the device W is not canonical


class WeightMoments(NamedTuple):
    """s0, s1, s2 of the weight matrix (``_g_moments``) and its number of rows."""

    s0: Any
    s1: Any
    s2: Any
    n: int


def _weight_moments(w: Any) -> WeightMoments:
    return w if isinstance(w, WeightMoments) else WeightMoments(*_g_moments(w), w.shape[0])


# ---------------------------------------------------------------------------------------------------------
# device plan
# ---------------------------------------------------------------------------------------------------------
class AutocorrPlan:
    """Device-resident weight matrix W (CSR) + loaded feature matrix: the object behind ``sqb_autocorr``.
    ``score(mode, row_perm)`` replaces ``morans_i(g, vals)`` / ``gearys_c(g, vals)``."""

    def __init__(self, g: spmatrix, ctx: Context | None = None):
        self._lib = load()
        self.ctx = ctx or default_context()
        g = as_csr(g)
        if g.shape[0] != g.shape[1]:
            raise ValueError(f"Expected a square weight matrix, found shape `{g.shape}`.")
        self.n = g.shape[0]
        wp = np.ascontiguousarray(g.indptr, dtype=np.int32)
        wi = np.ascontiguousarray(g.indices, dtype=np.int32)
        if g.data.dtype == np.float32:
            wd, wdt = np.ascontiguousarray(g.data), 0
        else:
            wd, wdt = np.ascontiguousarray(g.data, dtype=np.float64), 1
        h = C.c_void_p()
        check(self._lib.sqb_autocorr_create(self.ctx.handle, self.n, wi.size, wp.ctypes.data, wi.ctypes.data, wd.ctypes.data, wdt, C.byref(h)))
        self._h = h
        self.n_features = 0

    @classmethod
    def from_device(cls, graph: DevGraph, transformation: bool, ctx: Context | None = None) -> "AutocorrPlan | None":
        """Plan over a weight matrix already in GPU memory (``weight_graph_args`` of a torch ``sparse_csr`` or cupyx-style CSR with
        float32 / float64 values and canonical rows), read in place and never on the host or modified.  ``transformation``
        row-normalises W on the device like ``normalize(W, norm="l1", axis=1)``.  ``moments`` holds s0, s1, s2 of
        ``_g_moments`` of the normalised W, as numpy scalars of W's dtype.  Returns ``None`` when a row's column indices do
        not strictly increase, or when W holds NaN / infinite weights and ``transformation`` is set (sklearn rejects those):
        the caller then takes the host copy.  An index out of range or a bad indptr raise."""
        if graph.transposed:
            raise ValueError("Expected a CSR weight matrix.")
        code = {np.dtype(np.float32): 0, np.dtype(np.float64): 1}.get(graph.sparse.data.dtype)
        if code is None:
            raise TypeError(f"Device weight matrices of dtype `{graph.sparse.data.dtype}` are read on the host; use float32 or float64.")
        data = graph.sparse.data
        if len(data.shape) != 1 or data.shape[0] != graph.nnz or (graph.nnz > 1 and data.strides[0] != 1):
            raise ValueError(f"The weight matrix's values must be a contiguous 1-D array of `{graph.nnz}` entries.")
        self = cls.__new__(cls)
        self._h = None
        self._lib = load()
        self.ctx = ctx or default_context()
        self.n = graph.n
        self.n_features = 0
        h = C.c_void_p()
        mom = np.zeros(3, dtype=np.float64)
        rc = self._lib.sqb_autocorr_create_device(self.ctx.handle, graph.n, graph.nnz, graph.indptr, graph.indptr_bits, graph.indices or None,
                                                  graph.index_bits, graph.sparse.data.ptr or None, code, int(bool(transformation)),
                                                  graph.stream, mom.ctypes.data, C.byref(h))
        if rc == SQB_ERR_LAYOUT:
            return None
        check(rc)
        self._h = h
        t = graph.sparse.data.dtype.type
        self.moments = WeightMoments(t(mom[0]), t(mom[1]), t(mom[2]), graph.n)
        return self

    @property
    def w_info(self) -> tuple[int, int]:
        """``(format, s0_branch)`` of the plan's W: format 0 packed rows of 8 slots, 1 of 16, 2 CSR walk, 3 compact rows;
        s0_branch 0 = S0 summed exactly in parallel, 1 = on one ordered thread."""
        f, b = C.c_int(), C.c_int()
        check(self._lib.sqb_autocorr_w_info(self._h, C.byref(f), C.byref(b)))
        return f.value, b.value

    @staticmethod
    def _dt(a: np.ndarray) -> tuple[np.ndarray, int]:
        if a.dtype == np.float32:
            return np.ascontiguousarray(a), 0
        return np.ascontiguousarray(a, dtype=np.float64), 1  # ints, float16, float64 ... -> float64 like scanpy's astype

    def load(self, m: Any, *, obs_major: bool, cols: tuple[int, int] | None = None, col_map: np.ndarray | None = None) -> None:
        """``m``: observations x features if ``obs_major`` else features x observations; dense or scipy sparse, or resident
        in device memory (see :mod:`squidpy_b200._device`): then it is read in place on the device and never copied to the host.
        ``cols=(lo, hi)`` loads only features ``lo..hi`` (the shard of one rank): for CSR-by-observation input the slice is
        cut while the matrix is staged for the upload (``sqb_autocorr_load_csr_cols``), nothing is copied on the host.
        ``col_map`` (device input only, instead of ``cols``): int32 per input feature, its index among the loaded features
        or -1 to skip it."""
        n_feat = int(m.shape[1] if obs_major else m.shape[0])
        n_obs = int(m.shape[0] if obs_major else m.shape[1])
        if n_obs != self.n:
            raise ValueError(f"Expected `{self.n}` observations, found `{n_obs}`.")
        dev = device_matrix(m)
        if dev is not None:
            self._load_device(dev, obs_major, n_feat, cols, col_map)
            return
        if col_map is not None:
            raise ValueError("`col_map` applies to device-resident input only.")
        if cols is not None and tuple(cols) == (0, n_feat):
            cols = None
        if issparse(m):
            if m.format == "csc":  # CSC of (a x b) == CSR of (b x a): flip the orientation instead of converting
                m = m.T
                obs_major = not obs_major
            elif m.format != "csr":
                m = m.tocsr()
            # entry order inside a row does not matter and repeated entries are rejected by the device (no host pass over
            # the non-zeros); only the column-sliced upload needs ascending indices
            if cols is not None and obs_major:
                if not m.has_sorted_indices:
                    m = m.copy()
                    m.sort_indices()
                data, dt = self._dt(m.data)
                xp = np.ascontiguousarray(m.indptr, dtype=np.int64)
                xi = np.ascontiguousarray(m.indices, dtype=np.int32)
                check(self._lib.sqb_autocorr_load_csr_cols(self._h, xp.ctypes.data, xi.ctypes.data, data.ctypes.data, dt, n_feat, int(cols[0]), int(cols[1])))
                self.n_features = int(cols[1] - cols[0])
                return
            if cols is not None:
                m = m[cols[0] : cols[1]]  # features x observations: a row slice of the CSR is cheap
                n_feat = m.shape[0]
            data, dt = self._dt(m.data)
            xp = np.ascontiguousarray(m.indptr, dtype=np.int64)
            xi = np.ascontiguousarray(m.indices, dtype=np.int32)
            check(self._lib.sqb_autocorr_load_csr(self._h, xp.ctypes.data, xi.ctypes.data, data.ctypes.data, dt, int(obs_major), n_feat))
        else:
            a = np.asarray(m)
            if cols is not None:
                a = a[:, cols[0] : cols[1]] if obs_major else a[cols[0] : cols[1]]
                n_feat = cols[1] - cols[0]
            a, dt = self._dt(a)
            check(self._lib.sqb_autocorr_load_dense(self._h, a.ctypes.data, dt, int(obs_major), n_feat))
        self.n_features = int(n_feat)

    def _load_device(self, d: DevArray | DevSparse, obs_major: bool, n_feat: int, cols: tuple[int, int] | None,
                     col_map: np.ndarray | None) -> None:
        if col_map is None:
            lo, hi = cols if cols is not None else (0, n_feat)
            col_map, n_out, _ = feature_map(n_feat, np.arange(lo, hi))
        else:
            col_map = np.ascontiguousarray(col_map, dtype=np.int32)
            if col_map.shape != (n_feat,):
                raise ValueError(f"Expected `col_map` of length `{n_feat}`, found shape `{col_map.shape}`.")
            n_out = int(col_map.max(initial=-1)) + 1
        if n_out < 1:
            raise ValueError("No feature selected.")
        dev = array_device(d, pointer_device)
        if dev != self.ctx.device:
            raise ValueError(f"The matrix lives on cuda:{dev}, but this plan's context is on cuda:{self.ctx.device}.")
        stream = common_stream(d)
        if isinstance(d, DevSparse):
            # CSC of (a x b) == CSR of (b x a): the orientation flips instead of a conversion
            layout = int(obs_major) if d.format == "csr" else int(not obs_major)
            check(self._lib.sqb_autocorr_load_csr_device(self._h, d.indptr.ptr, index_bits(d.indptr, "indptr"), d.indices.ptr,
                                                         index_bits(d.indices, "indices"), d.data.ptr, dtype_code(d.data), layout, n_feat,
                                                         col_map.ctypes.data, n_out, stream))
        else:
            if len(d.shape) != 2:
                raise ValueError(f"Expected a 2-D device array, found shape `{d.shape}`.")
            check(self._lib.sqb_autocorr_load_dense_device(self._h, d.ptr, dtype_code(d), d.shape[0], d.shape[1], d.strides[0], d.strides[1],
                                                           int(obs_major), col_map.ctypes.data, n_out, stream))
        self.n_features = n_out

    def run_async(self, mode: SpatialAutocorr | str, row_perm: np.ndarray | None = None) -> None:
        mode = SpatialAutocorr(mode)
        rp = None if row_perm is None else np.ascontiguousarray(row_perm, dtype=np.int64)
        check(self._lib.sqb_autocorr_run_async(self._h, 0 if mode == SpatialAutocorr.MORAN else 1, None if rp is None else rp.ctypes.data))

    def download(self) -> np.ndarray:
        out = np.empty(self.n_features, dtype=np.float64)
        check(self._lib.sqb_autocorr_download(self._h, out.ctypes.data))
        return out

    def score(self, mode: SpatialAutocorr | str, row_perm: np.ndarray | None = None) -> np.ndarray:
        self.run_async(mode, row_perm)
        return self.download()

    def score_perms(self, mode: SpatialAutocorr | str, row_perms: np.ndarray) -> np.ndarray:
        """``_score_helper`` (``_ppatterns.py:258-280``) for a stack of permutations: ``row_perms`` is (P, n) with row p the
        ``idx_shuffle`` of permutation p; returns float64 (P, n_features).  X stays on the device."""
        mode = SpatialAutocorr(mode)
        rp = np.ascontiguousarray(np.atleast_2d(row_perms), dtype=np.int64)
        if rp.shape[1] != self.n:
            raise ValueError(f"Expected permutations of length `{self.n}`, found `{rp.shape[1]}`.")
        out = np.empty((rp.shape[0], self.n_features), dtype=np.float64)
        check(self._lib.sqb_autocorr_run_perms(self._h, 0 if mode == SpatialAutocorr.MORAN else 1, rp.ctypes.data, rp.shape[0], out.ctypes.data))
        return out

    def close(self) -> None:
        if self._h is not None:
            self._lib.sqb_autocorr_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


# ---------------------------------------------------------------------------------------------------------
# spatial_autocorr
# ---------------------------------------------------------------------------------------------------------
def spatial_autocorr(
    adata: Any,
    connectivity_key: str = Key.obsp.spatial_conn(),
    genes: str | int | Sequence[str] | Sequence[int] | None = None,
    mode: SpatialAutocorr | Literal["moran", "geary"] = "moran",
    transformation: bool = True,
    n_perms: int | None = None,
    two_tailed: bool = False,
    corr_method: str | None = "fdr_bh",
    attr: Literal["obs", "X", "obsm"] = "X",
    layer: str | None = None,
    seed: int | None = None,
    use_raw: bool = False,
    copy: bool = False,
    n_jobs: int | None = None,
    backend: str = "loky",
    show_progress_bar: bool = True,
    *,
    table_key: str | None = None,
    device: int | None = None,
) -> pd.DataFrame | None:
    """Calculate Global Autocorrelation Statistic (Moran's I or Geary's C) — see module docstring.

    Returns / writes ``adata.uns['moranI' | 'gearyC']``: DataFrame indexed by feature with columns ``I``|``C``,
    ``pval_norm``, ``var_norm``, (with ``n_perms``) ``pval_z_sim``, ``pval_sim``, ``var_sim``, and
    ``{pval}_{corr_method}``; sorted by the statistic.  Under ``torch.distributed`` the features are sharded over
    ranks (one all-gather of the scores).

    ``adata.X`` / ``layers[layer]`` / ``raw.X`` / ``obsm[layer]`` may be resident in device memory (cupy / cupyx.scipy.sparse,
    torch CUDA tensors, anything exposing ``__cuda_array_interface__``): the features are then selected and scored on the
    array's own device (``device`` must match it), and the matrix is never copied to the host.  A device-resident
    ``obsp[connectivity_key]`` in CSR layout with float32 / float64 values and canonical rows (strictly increasing column
    indices: what ``spatial_neighbors_*`` export) is read in place on its own device: its row normalisation, S0, column sums
    and the moments of the p-values are computed there, equal bit for bit to the host computation, and the caller's graph is
    neither modified nor copied to the host.  ``device`` must match that device, and a device X must live on it too.  Any
    other device graph (CSC, integer / bool / float16 values, strided or mis-sized arrays, unsorted or repeated column
    indices, NaN / infinite weights to normalise, dense) is copied to the host once and handled as a host graph."""
    adata = extract_adata_if_sdata(adata, table_key=table_key)
    assert_connectivity_key(adata, connectivity_key)

    # ---- feature matrix, observations x features (the reference builds the transpose, :154-194) ----
    def select_genes(genes):  # the feature list and its order, for host and device matrices alike
        if genes is None:
            if "highly_variable" in adata.var:
                genes = adata.var_names[np.asarray(adata.var["highly_variable"], dtype=bool)].values
            else:
                genes = adata.var_names.values
        elif isinstance(genes, str):
            genes = [genes]
        if use_raw:
            if adata.raw is None:
                raise AttributeError("No `.raw` attribute found. Try specifying `use_raw=False`.")
            genes = list(set(genes) & set(adata.raw.var_names))
        return genes

    def extract_X(genes):
        if not use_raw:
            if len(genes) == adata.shape[1] and np.array_equal(np.asarray(genes), np.asarray(adata.var_names)):
                # all variables in their own order: the subset is the matrix itself (the reference's adata[:, genes] copies it
                # on the host; at 4e8 non-zeros that copy alone costs seconds)
                return (adata.X if layer is None else adata.layers[layer]), genes
            subset = adata[:, genes]
            return (subset.X if layer is None else subset.layers[layer]), genes
        return adata.raw[:, genes].X, genes

    def extract_obs(cols):
        if cols is None:
            df = adata.obs.select_dtypes(include=np.number)
            return df.to_numpy(), df.columns
        if isinstance(cols, str):
            cols = [cols]
        return adata.obs[cols].to_numpy(), cols

    def obsm_columns(ixs):
        assert_key_in_adata(adata, layer, attr="obsm")
        if ixs is None:
            ixs = list(np.arange(adata.obsm[layer].shape[1]))
        return list(np.ravel([ixs]))

    # device-resident matrix: `src` (every feature) and the column `positions` of the selected ones; X is not touched here
    src, positions = None, None
    if attr == "X":
        genes = select_genes(genes)
        src = adata.raw.X if use_raw else (adata.X if layer is None else adata.layers[layer])
        if device_matrix(src) is None:
            src = None
            mat, index = extract_X(genes)
        else:
            index = genes
            positions = var_positions(adata.raw.var_names if use_raw else adata.var_names, genes)
    elif attr == "obs":
        mat, index = extract_obs(genes)
    elif attr == "obsm":
        index = obsm_columns(genes)
        src = adata.obsm[layer]
        if device_matrix(src) is None:
            src = None
            mat = adata.obsm[layer][:, index]
        else:
            positions = np.asarray(index, dtype=np.int64)
    else:
        raise NotImplementedError(f"Extracting from `adata.{attr}` is not yet implemented.")

    mode = SpatialAutocorr(mode)
    params: dict[str, Any] = {"mode": mode.s, "transformation": transformation, "two_tailed": two_tailed}
    if mode == SpatialAutocorr.MORAN:
        params.update(stat="I", expected=-1.0 / (adata.shape[0] - 1), ascending=False)
    else:
        params.update(stat="C", expected=1.0, ascending=True)

    g_src = adata.obsp[connectivity_key]
    w_dev = device_matrix(g_src)
    # a device CSR with float values in contiguous arrays is read where it lives; everything else is copied to the host (sklearn /
    # scipy there)
    w_graph = weight_graph_args(w_dev, adata.shape[0])

    def host_w():
        g = g_src.copy() if w_dev is None else to_host_matrix(g_src)
        if transformation:  # row-normalise in place, dtype preserved (float32 stays float32), :212-214
            from sklearn.preprocessing import normalize

            normalize(g, norm="l1", axis=1, copy=False)
        return g

    g = None if w_graph is not None else host_w()

    start = time.perf_counter()
    n_feat = mat.shape[1] if src is None else len(positions)
    rank, ws = world()
    lo, hi = shard_range(n_feat, rank, ws)
    expand = None  # device input: scores of the shard = loaded scores[expand] (duplicate features are loaded once)
    if w_graph is not None:  # the plan lives on W's device
        on_w = array_device(w_dev, pointer_device)
        if device is not None and int(device) != on_w:
            raise ValueError(f"`device={device}` does not match the device of the weight matrix, cuda:{on_w}.")
        device = on_w
    if src is not None:
        on = array_device(device_matrix(src), pointer_device)
        if w_graph is not None and on != device:
            raise ValueError(f"The feature matrix lives on cuda:{on}, but the weight matrix on cuda:{device}.")
        if device is not None and int(device) != on:
            raise ValueError(f"`device={device}` does not match the device of the feature matrix, cuda:{on}.")
        device = on
    ctx = default_context(device)
    logg.info("Calculating %s's statistic for `%s` permutations on cuda:%d (rank %d/%d, features %d..%d)", mode, n_perms, ctx.device, rank, ws, lo, hi)
    with ctx.lock:
        plan = None
        if w_graph is not None:
            plan = AutocorrPlan.from_device(w_graph, transformation, ctx)
            if plan is None:  # a row that is not canonical, or non-finite weights to normalise: the host copy handles it as before
                g = host_w()
        if plan is None:
            plan = AutocorrPlan(g, ctx)
        weights = plan.moments if g is None else g
        n_obs = plan.n
        try:
            if hi > lo and src is not None:
                col_map, _, expand = feature_map(src.shape[1], positions, lo, hi)
                plan.load(src, obs_major=True, col_map=col_map)
                score_local = plan.score(mode)[expand]
            elif hi > lo:
                plan.load(mat, obs_major=True, cols=(lo, hi))
                score_local = plan.score(mode)
            else:
                score_local = np.empty(0, np.float64)
            score = all_gather_rows(score_local, n_feat)
            score_perms = None
            if n_perms is not None:
                assert_positive(n_perms, name="n_perms")
                generators = spawn_generators(shared_seed(seed), int(n_perms))
                sp_local = np.empty((int(n_perms), hi - lo), dtype=np.float64)
                batch = max(1, min(32, (256 << 20) // (8 * n_obs)))  # <= 256 MB of int64 permutations per device call
                from concurrent.futures import ThreadPoolExecutor

                def draw(p0):  # idx_shuffle of _score_helper (:258-280) for one batch; numpy releases the GIL while it shuffles
                    return np.stack([generators[p].permutation(n_obs) for p in range(p0, min(p0 + batch, int(n_perms)))])

                starts = list(range(0, int(n_perms), batch))
                with ThreadPoolExecutor(max_workers=1) as pool:  # the next batch is drawn while the device scores this one
                    nxt = pool.submit(draw, starts[0])
                    for k, p0 in enumerate(starts):
                        idx = nxt.result()
                        if k + 1 < len(starts):
                            nxt = pool.submit(draw, starts[k + 1])
                        if hi > lo:
                            sp = plan.score_perms(mode, idx)
                            sp_local[p0 : p0 + idx.shape[0]] = sp if expand is None else sp[:, expand]
                score_perms = np.ascontiguousarray(all_gather_rows(np.ascontiguousarray(sp_local.T), n_feat).T)
        finally:
            plan.close()

    with np.errstate(divide="ignore", invalid="ignore"):
        pval_results = _p_value_calc(score, score_perms, weights, params)

    df = pd.DataFrame({str(params["stat"]): score, **pval_results}, index=index)
    if corr_method is not None:
        for pv in [c for c in df.columns if "pval" in c]:
            df[f"{pv}_{corr_method}"] = _multipletests(df[pv].values, method=corr_method)
    df.sort_values(by=params["stat"], ascending=params["ascending"], inplace=True)

    if copy:
        logg.info("Finish (%.3fs)", time.perf_counter() - start)
        return df
    _save_data(adata, attr="uns", key=str(params["mode"]) + str(params["stat"]), data=df, time_start=start)
    return None


def _multipletests(pvals: np.ndarray, method: str) -> np.ndarray:
    """p-value adjustment (``statsmodels.stats.multitest.multipletests(pvals, alpha=0.05, method=...)[1]``,
    used at ``_ppatterns.py:242-245``).  ``fdr_bh`` (the default), ``fdr_by``, ``bonferroni``, ``holm`` and ``sidak``
    are implemented here because statsmodels is not a dependency; anything else defers to statsmodels if present."""
    p = np.asarray(pvals, dtype=np.float64)
    n = p.size
    if method in ("fdr_bh", "fdr_by"):
        order = np.argsort(p)
        ps = p[order]
        ecdf = np.arange(1, n + 1) / float(n)
        if method == "fdr_by":
            ecdf = ecdf / np.sum(1.0 / np.arange(1, n + 1))
        corrected = ps / ecdf
        corrected = np.minimum.accumulate(corrected[::-1])[::-1]
        corrected[corrected > 1] = 1
        out = np.empty(n)
        out[order] = corrected
        return out
    if method == "bonferroni":
        return np.minimum(p * n, 1.0)
    if method == "sidak":
        return 1.0 - np.power(1.0 - p, n)
    if method == "holm":
        order = np.argsort(p)
        adj = np.maximum.accumulate(p[order] * np.arange(n, 0, -1))
        out = np.empty(n)
        out[order] = np.minimum(adj, 1.0)
        return out
    try:
        from statsmodels.stats.multitest import multipletests
    except ImportError as e:
        raise NotImplementedError(f"`corr_method={method!r}` needs statsmodels, which is not installed.") from e
    return multipletests(p, alpha=0.05, method=method)[1]


def _p_value_calc(score: np.ndarray, sims: np.ndarray | None, weights: Any, params: dict[str, Any]) -> dict[str, Any]:
    """p-values of the autocorrelation scores (``_ppatterns.py:443-498``): analytic (normality) and, with
    permutations, simulation based.  ``weights``: the weight matrix, or its ``WeightMoments``."""
    p_norm, var_norm = _analytic_pval(score, weights, params)
    results = {"pval_norm": p_norm, "var_norm": var_norm}
    if sims is None:
        return results
    n_perms = sims.shape[0]
    large_perm = (sims >= score).sum(axis=0)
    flip = (n_perms - large_perm) < large_perm  # two-sided tail selection
    large_perm[flip] = n_perms - large_perm[flip]
    p_sim = (large_perm + 1) / (n_perms + 1)
    e_score_sim = sims.sum(axis=0) / n_perms
    se_score_sim = sims.std(axis=0)
    z_sim = (score - e_score_sim) / se_score_sim
    p_z_sim = np.empty(z_sim.shape)
    pos = z_sim > 0
    p_z_sim[pos] = 1 - stats.norm.cdf(z_sim[pos])
    p_z_sim[z_sim <= 0] = stats.norm.cdf(z_sim[z_sim <= 0])
    results["pval_z_sim"] = p_z_sim
    results["pval_sim"] = p_sim
    results["var_sim"] = np.var(sims, axis=0)
    return results


def _analytic_pval(score: np.ndarray, g: Any, params: dict[str, Any]) -> tuple[np.ndarray, float]:
    """Normality-assumption variance and p-value (Cliff & Ord 1981; ``_ppatterns.py:501-538``).  ``g``: the weight matrix,
    or its ``WeightMoments``."""
    s0, s1, s2, n = _weight_moments(g)
    s02 = s0 * s0
    if params["mode"] == SpatialAutocorr.GEARY.s:
        v_score = ((2 * s1 + s2) * (n - 1) - 4 * s02) / (2 * (n + 1) * s02)
    elif params["mode"] == SpatialAutocorr.MORAN.s:
        n2 = n * n
        v_num = n2 * s1 - n * s2 + 3 * s02
        v_den = (n - 1) * (n + 1) * s02
        v_score = v_num / v_den - (1.0 / (n - 1)) ** 2
    else:
        raise AssertionError(f"Unexpected mode `{params['mode']}`.")
    se_score = v_score ** (1 / 2.0)
    z_norm = (score - params["expected"]) / se_score
    p_norm = np.empty(score.shape)
    pos = z_norm > 0
    p_norm[pos] = 1 - stats.norm.cdf(z_norm[pos])
    p_norm[z_norm <= 0] = stats.norm.cdf(z_norm[z_norm <= 0])
    if params["two_tailed"]:
        p_norm *= 2.0
    return p_norm, v_score


def _g_moments(w: Any) -> tuple[float, float, float]:
    """s0, s1, s2 of the weight matrix (pysal definitions; ``_ppatterns.py:541-559``).  Evaluated in W's own dtype
    (float32 for a row-normalised squidpy graph), which is what the reference's p-values are built on."""
    s0 = w.sum()
    t = w.transpose() + w
    t2 = t.multiply(t) if isinstance(t, spmatrix) or issparse(t) else t * t
    s1 = t2.sum() / 2.0
    s2array = np.array(w.sum(1) + w.sum(0).transpose()) ** 2
    s2 = s2array.sum()
    return s0, s1, s2


# ---------------------------------------------------------------------------------------------------------
# co_occurrence
# ---------------------------------------------------------------------------------------------------------
def cooc_counts(x: np.ndarray, y: np.ndarray, thresholds: np.ndarray, labs: np.ndarray, k: int, *, use_fma: bool = True,
                ctx: Context | None = None, shard: tuple[int, int] = (0, 1)) -> np.ndarray:
    """``_occur_count`` (``_ppatterns.py:283-310``) on the GPU: int64 (k, k, L) cumulative ordered-pair counts.
    Thresholds need not be sorted (each radius is independent in the reference); they are sorted for the device and
    the result is mapped back."""
    lib = load()
    ctx = ctx or default_context()
    x = np.ascontiguousarray(x, dtype=np.float32)
    y = np.ascontiguousarray(y, dtype=np.float32)
    labs = np.ascontiguousarray(labs, dtype=np.int32)
    thr = np.ascontiguousarray(thresholds, dtype=np.float32)
    order = np.argsort(thr, kind="stable")
    thr_sorted = np.ascontiguousarray(thr[order])
    out = np.empty((k, k, thr.size), dtype=np.int64)
    check(lib.sqb_cooc_counts(ctx.handle, x.ctypes.data, y.ctypes.data, x.size, labs.ctypes.data, int(k), thr_sorted.ctypes.data,
                              thr.size, int(use_fma), int(shard[0]), int(shard[1]), out.ctypes.data))
    if not np.array_equal(order, np.arange(thr.size)):
        inv = np.empty_like(order)
        inv[order] = np.arange(thr.size)
        out = np.ascontiguousarray(out[:, :, inv])
    return out


def _co_occurrence_helper(v_x: np.ndarray, v_y: np.ndarray, v_radium: np.ndarray, labs: np.ndarray, *, ctx: Context | None = None):
    """``_co_occurrence_helper`` (``_ppatterns.py:313-358``): GPU counts + the conditional-probability ratio
    ``occ[i,c,r] = (counts[c,i,r] / row_sums[c,r]) / (row_sums[i,r] / totals[r])``."""
    labs_unique, labs_dense = np.unique(labs, return_inverse=True)  # present codes -> 0..k-1 (identity when all present)
    k = len(labs_unique)
    l_val = len(v_radium) - 1
    thresholds = (v_radium[1:]) ** 2
    rank, ws = world()
    counts = cooc_counts(v_x, v_y, thresholds, labs_dense.astype(ip), k, ctx=ctx, shard=(rank, ws))
    counts = all_reduce_sum(counts)
    occ_prob = np.zeros((k, k, l_val), dtype=np.float64)
    row_sums = counts.sum(axis=0)
    totals = row_sums.sum(axis=0)
    with np.errstate(divide="ignore", invalid="ignore"):
        probs = row_sums / totals[None, :]  # (k, L)
        cond = counts / row_sums[:, None, :]  # cond[c, i, r] = counts[c,i,r] / row_sums[c,r]
        ratio = np.transpose(cond, (1, 0, 2)) / probs[:, None, :]  # [i, c, r]
    ok = (probs[:, None, :] != 0.0) & (row_sums[None, :, :] != 0.0)
    occ_prob[ok] = ratio[ok]
    return occ_prob, counts


def co_occurrence(
    adata: Any,
    cluster_key: str,
    spatial_key: str = Key.obsm.spatial,
    interval: int | np.ndarray = 50,
    copy: bool = False,
    *,
    table_key: str | None = None,
    device: int | None = None,
    **deprecated: Any,
) -> tuple[np.ndarray, np.ndarray] | None:
    """Compute co-occurrence probability of clusters (``_ppatterns.py:361-428``).

    Returns ``(occ float64[k,k,L], interval float32[L+1])`` if ``copy=True``; otherwise writes
    ``adata.uns[f'{cluster_key}_co_occurrence'] = {'occ', 'interval'}``.  ``n_splits``, ``n_jobs``, ``backend`` and
    ``show_progress_bar`` are accepted and ignored with a ``FutureWarning`` like in the reference (:362)."""
    for kname in list(deprecated):
        if kname in ("n_splits", "n_jobs", "backend", "show_progress_bar"):
            warnings.warn(
                f"Parameter `{kname}` of `co_occurrence()` is deprecated and has no effect. It will be removed in squidpy v1.10.0.",
                FutureWarning,
                stacklevel=2,
            )
            deprecated.pop(kname)
    if deprecated:
        raise TypeError(f"co_occurrence() got an unexpected keyword argument '{next(iter(deprecated))}'")

    adata = extract_adata_if_sdata(adata, table_key=table_key)
    assert_categorical_obs(adata, key=cluster_key)
    assert_spatial_basis(adata, key=spatial_key)

    spatial = np.asarray(on_host(adata.obsm[spatial_key])).astype(fp)
    labs, _ = category_codes(adata.obs[cluster_key], dtype=ip)

    if isinstance(interval, int):
        thresh_min, thresh_max = _find_min_max(spatial)
        interval = np.linspace(thresh_min, thresh_max, num=interval, dtype=fp)
    else:
        interval = np.array(sorted(interval), dtype=fp, copy=True)
    if len(interval) <= 1:
        raise ValueError(f"Expected interval to be of length `>= 2`, found `{len(interval)}`.")

    start = time.perf_counter()
    logg.info("Calculating co-occurrence probabilities for `%d` intervals", len(interval))
    out, _ = _co_occurrence_helper(spatial[:, 0], spatial[:, 1], interval, labs, ctx=default_context(device))

    if copy:
        logg.info("Finish (%.3fs)", time.perf_counter() - start)
        return out, interval
    _save_data(adata, attr="uns", key=Key.uns.co_occurrence(cluster_key), data={"occ": out, "interval": interval}, time_start=start)
    return None


def _find_min_max(spatial: np.ndarray) -> tuple[float, float]:
    """Default radius range (``_ppatterns.py:431-440``): smallest = distance between the two points with the smallest
    coordinate sum, largest = half the distance between the extreme coordinate sums (sklearn pairwise_distances on
    float32, like the reference)."""
    from sklearn.metrics import pairwise_distances

    coord_sum = np.sum(spatial, axis=1)
    min_idx, min_idx2 = np.argpartition(coord_sum, 2)[:2]
    max_idx = np.argmax(coord_sum)
    thres_max = pairwise_distances(spatial[min_idx, :].reshape(1, -1), spatial[max_idx, :].reshape(1, -1))[0, 0] / 2.0
    thres_min = pairwise_distances(spatial[min_idx, :].reshape(1, -1), spatial[min_idx2, :].reshape(1, -1))[0, 0]
    return thres_min.astype(fp), thres_max.astype(fp)
