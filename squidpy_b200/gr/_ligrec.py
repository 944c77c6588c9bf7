"""``ligrec`` — receptor-ligand permutation test (CellPhoneDB) with the permutations on an H100; drop-in for the
explicit-interactions use of ``squidpy.gr.ligrec`` (``src/squidpy/gr/_ligrec.py``).

What runs where
  * per permutation: shuffle the cluster labels with numpy's generator ``p`` of ``spawn_generators(seed, n_perms)`` (exact
    device replay, shared with nhood_enrichment), re-form the per-cluster mean of every gene, compare
    ``mean[a, g0] + mean[b, g1] > observed`` for every (interaction, cluster pair) — ``sqb_ligrec_counts``, replacing the
    numba kernel ``_score_permutations`` (``_ligrec.py:616-676``) with the same float64 operation order;
  * once per call, on the host with the reference's own pandas expressions (so that the observed means the decisions are
    taken against are bit-identical): group means, expression-fraction mask, validity, result frames, FDR
    (``_analysis`` ``_ligrec.py:679-776``, ``PermutationTest.test`` ``:230-370``).
Interactions must be given (DataFrame / dict / sequences); the reference's ``interactions=None`` downloads them from
omnipath, which needs network access and is not replicated.
"""

from __future__ import annotations

import ctypes as C
import time
from collections.abc import Iterable, Mapping
from itertools import product
from typing import Any, NamedTuple

import numpy as np
import pandas as pd

from .._constants import ComplexPolicy, CorrAxis, Key
from .._device import device_matrix
from .._dist import all_reduce_sum, shard_range, shared_seed, world
from .._lib import Context, check, default_context, load
from .._rng import spawn_states
from .._validators import assert_categorical_obs, assert_positive, extract_adata_if_sdata
from ._gather import OBS_MAJOR, Gathered, device_context
from ._utils import _save_data, logg

__all__ = ["ligrec", "ligrec_analysis", "ligrec_analysis_device", "TempResult"]

SOURCE = "source"
TARGET = "target"


class TempResult(NamedTuple):
    """``(n_interactions, n_interaction_clusters)`` means and p-values (``_ligrec.py:48-54``)."""

    means: np.ndarray
    pvalues: np.ndarray


def ligrec_analysis(data: pd.DataFrame, interactions: np.ndarray, interaction_clusters: np.ndarray, threshold: float = 0.1,
                    n_perms: int = 1000, seed: int | None = None, *, ctx: Context | None = None) -> TempResult:
    """``_analysis`` (``_ligrec.py:679-776``): ``data`` has one integer-named column per gene plus a categorical column
    ``'clusters'`` whose categories are ``0 .. n_cls-1``; ``interactions`` holds column positions, ``interaction_clusters``
    cluster codes.
    Under an initialised ``torch.distributed`` process group (one process per GPU) the permutations are sharded over the ranks
    and the permutation counts summed once over them; every rank gets the full result."""
    clustering = np.array(data["clusters"].values, dtype=np.int32)
    data = data.astype({c: np.float64 for c in data.columns if c != "clusters"})
    groups = data.groupby("clusters", observed=True)
    mean_obs = groups.mean().values  # (n_clusters, n_genes): pandas' compensated group mean, the reference value
    mask = groups.apply(lambda c: ((c > 0).astype(np.int64).sum() / len(c)) >= threshold).values
    cluster_sizes = groups.size().values.astype(np.float64)
    data_arr = np.array(data[data.columns.difference(["clusters"])].values, dtype=np.float64, order="C")
    inter, cpairs, inv_counts, valid, res_means = _decisions(mean_obs, mask, cluster_sizes, interactions, interaction_clusters)

    n_cells, n_genes = data_arr.shape
    ctx = ctx or default_context()

    def counts_call(lib, h, inv, mean_c, valid_u8, counts):
        check(lib.sqb_ligrec_counts(h, data_arr.ctypes.data, n_genes, inv.ctypes.data, mean_c.ctypes.data, inter.ctypes.data, inter.shape[0],
                                    cpairs.ctypes.data, cpairs.shape[0], valid_u8.ctypes.data, counts.ctypes.data))

    return _permutation_test(ctx, clustering, mean_obs.shape[0], inter, cpairs, inv_counts, mean_obs, valid, res_means, n_perms, seed, counts_call)


def _decisions(mean_obs: np.ndarray, mask: np.ndarray, cluster_sizes: np.ndarray, interactions: np.ndarray, interaction_clusters: np.ndarray):
    """From the observed per-cluster means, the expression-fraction mask and the cluster sizes: the interaction / cluster-pair
    arrays for the library, ``1 / size``, which (interaction, cluster pair) cells are tested, and the result means
    (``_analysis``, ``_ligrec.py:700-740``)."""
    inv_counts = 1.0 / np.maximum(cluster_sizes, 1)
    inter = np.ascontiguousarray(interactions, dtype=np.int32)
    cpairs = np.ascontiguousarray(interaction_clusters, dtype=np.int32)
    rec, lig, c1, c2 = inter[:, 0], inter[:, 1], cpairs[:, 0], cpairs[:, 1]
    m_rec = mean_obs[c1, :][:, rec].T
    m_lig = mean_obs[c2, :][:, lig].T
    nonzero = (m_rec > 0) & (m_lig > 0)
    valid = nonzero & mask[c1, :][:, rec].T & mask[c2, :][:, lig].T
    res_means = np.where(nonzero, (m_rec + m_lig) / 2.0, 0.0)
    return inter, cpairs, inv_counts, valid, res_means


def _permutation_test(ctx: Context, clustering: np.ndarray, n_cls: int, inter: np.ndarray, cpairs: np.ndarray, inv_counts: np.ndarray,
                      mean_obs: np.ndarray, valid: np.ndarray, res_means: np.ndarray, n_perms: int, seed: int | None, counts_call) -> TempResult:
    """The permutation counts on a graph-less nhood handle whose base labels are ``clustering``; ``counts_call(lib, h, inv_counts,
    mean_obs, valid_u8, counts)`` runs the counting entry point on the expression matrix of the caller's choice.

    Under an initialised ``torch.distributed`` process group rank ``r`` counts only the permutations ``shard_range(n_perms, r,
    world)`` (generators of one family: ``seed=None`` is drawn once on rank 0) and the int64 counts are summed over the ranks in
    one all-reduce.  Integer sums are exact, so every rank gets the single-process result bit for bit."""
    n_cells = clustering.shape[0]
    counts = np.zeros((inter.shape[0], cpairs.shape[0]), dtype=np.int64)
    rank, ws = world()
    lo, hi = shard_range(int(n_perms), rank, ws)
    seed = shared_seed(seed)
    logg.info("Counting ligrec permutations on cuda:%d (rank %d/%d, permutations %d..%d)", ctx.device, rank, ws, lo, hi)
    if hi > lo:  # more ranks than permutations: this rank adds zeros (the handle refuses an empty upload)
        lib = load()
        valid_u8 = np.ascontiguousarray(valid, dtype=np.uint8)
        mean_c = np.ascontiguousarray(mean_obs, dtype=np.float64)
        with ctx.lock:
            h = C.c_void_p()
            empty_ptr = np.zeros(n_cells + 1, dtype=np.uint32)
            # a graph-less handle: only the label shuffle of the nhood machinery is used (n_cls >= 2 is asserted by the caller)
            check(lib.sqb_nhood_create(ctx.handle, n_cells, 0, empty_ptr.ctypes.data, None, max(n_cls, 2), C.byref(h)))
            try:
                lab = np.ascontiguousarray(clustering, dtype=np.uint32)
                check(lib.sqb_nhood_set_base(h, lab.ctypes.data, None, 0))
                states = spawn_states(seed, int(n_perms), lo, hi)
                check(lib.sqb_nhood_permute_upload(h, states.ctypes.data, states.shape[0]))
                counts_call(lib, h, inv_counts, mean_c, valid_u8, counts)
            finally:
                lib.sqb_nhood_destroy(h)
    counts = all_reduce_sum(counts)
    pvalues = counts.astype(np.float64) / n_perms
    pvalues[~valid] = np.nan
    return TempResult(means=res_means, pvalues=pvalues)


def ligrec_analysis_device(x: Gathered, clustering: np.ndarray, n_cls: int, interactions: np.ndarray, interaction_clusters: np.ndarray,
                           threshold: float = 0.1, n_perms: int = 1000, seed: int | None = None) -> TempResult:
    """``ligrec_analysis`` on a matrix gathered on the device (observations x genes, float64, NaN written as 0): cluster
    ``clustering[i]`` in ``[0, n_cls)`` for observation ``i``, every cluster present.  The observed means are pandas' group
    means bit for bit (``sqb_ligrec_observed``), so the result equals ``ligrec_analysis`` on the same values.
    Under an initialised ``torch.distributed`` process group (one process per GPU) the permutations are sharded over the ranks
    and the permutation counts summed once over them; every rank gets the full result."""
    lib = load()
    ctx = x.ctx
    codes = np.ascontiguousarray(clustering, dtype=np.int32)
    mean_obs = np.empty((n_cls, x.n_genes), dtype=np.float64)
    npos = np.empty((n_cls, x.n_genes), dtype=np.int64)
    sizes = np.empty(n_cls, dtype=np.int64)
    with ctx.lock:
        check(lib.sqb_ligrec_observed(x.handle, codes.ctypes.data, int(n_cls), mean_obs.ctypes.data, npos.ctypes.data, sizes.ctypes.data))
    cluster_sizes = sizes.astype(np.float64)
    mask = (npos / cluster_sizes[:, None]) >= threshold  # == ((c > 0).sum() / len(c)) >= threshold of every group
    inter, cpairs, inv_counts, valid, res_means = _decisions(mean_obs, mask, cluster_sizes, interactions, interaction_clusters)

    def counts_call(lib, h, inv, mean_c, valid_u8, counts):
        check(lib.sqb_ligrec_counts_dense(h, x.handle, inv.ctypes.data, mean_c.ctypes.data, inter.ctypes.data, inter.shape[0], cpairs.ctypes.data,
                                          cpairs.shape[0], valid_u8.ctypes.data, counts.ctypes.data))

    return _permutation_test(ctx, codes, n_cls, inter, cpairs, inv_counts, mean_obs, valid, res_means, n_perms, seed, counts_call)


# ---------------------------------------------------------------------------------------------------------
# host glue: interactions / complexes / result frames
# ---------------------------------------------------------------------------------------------------------
def _as_interaction_frame(interactions: Any) -> pd.DataFrame:
    if interactions is None:
        raise NotImplementedError("`interactions=None` fetches the interactions from omnipath (network access); pass them explicitly.")
    if isinstance(interactions, Mapping):
        interactions = pd.DataFrame(interactions)
    if isinstance(interactions, pd.DataFrame):
        for col in (SOURCE, TARGET):
            if col not in interactions.columns:
                raise KeyError(f"Column `{col!r}` is not in `interactions`.")
        df = interactions.copy()
    elif isinstance(interactions, Iterable):
        items = tuple(interactions)
        if not len(items):
            raise ValueError("No interactions were specified.")
        if isinstance(items[0], str):
            items = list(product(items, repeat=2))
        elif len(items) == 2:
            items = tuple(zip(*items, strict=False))
        if not all(len(i) == 2 for i in items):
            raise ValueError("Not all interactions are of length `2`.")
        df = pd.DataFrame(items, columns=[SOURCE, TARGET])
    else:
        raise TypeError(f"Expected either a `pandas.DataFrame`, `dict` or `iterable`, found `{type(interactions).__name__}`")
    if df.empty:
        raise ValueError("The interactions are empty")
    return df


def _resolve_complexes(df: pd.DataFrame, data: pd.DataFrame, policy: ComplexPolicy) -> pd.DataFrame:
    """``_filter_interactions_complexes`` (``_ligrec.py:389-451``): ``'A_B_C'`` names a protein complex."""
    if policy == ComplexPolicy.MIN:
        def pick(name):
            if name is None:
                return None
            if "_" not in name:
                return name
            parts = [c for c in name.split("_") if c in data.columns]
            if not parts:
                return None
            if len(parts) == 1:
                return parts[0]
            means = data[parts].mean()
            return str(means.index[means.argmin()])  # the least expressed component, like CellPhoneDB

        df[SOURCE] = df[SOURCE].apply(pick)
        df[TARGET] = df[TARGET].apply(pick)
        return df
    if policy == ComplexPolicy.ALL:
        src = df.pop(SOURCE).apply(lambda s: str(s).split("_")).explode()
        src.name = SOURCE
        tgt = df.pop(TARGET).apply(lambda s: str(s).split("_")).explode()
        tgt.name = TARGET
        df = pd.merge(df, src, how="left", left_index=True, right_index=True)
        return pd.merge(df, tgt, how="left", left_index=True, right_index=True)
    raise NotImplementedError(f"Complex policy {policy!r} is not implemented.")


def _multipletests(p: np.ndarray, method: str, alpha: float) -> np.ndarray:
    from ._ppatterns import _multipletests as mt

    return mt(p, method)


def _fdr_correct(pvals: pd.DataFrame, corr_method: str, corr_axis: CorrAxis, alpha: float) -> pd.DataFrame:
    """``_fdr_correct`` (``_ligrec.py:57-90``): NaNs (untested pairs) count as 1 during the correction and stay NaN."""
    def fdr(col: pd.Series):
        q = _multipletests(np.nan_to_num(col.values, copy=True, nan=1.0), corr_method, alpha)
        q[np.isnan(col.values)] = np.nan
        return pd.arrays.SparseArray(q, dtype=q.dtype, fill_value=np.nan)

    if corr_axis == CorrAxis.CLUSTERS:
        pvals = pvals.apply(fdr)  # clusters are in columns
    elif corr_axis == CorrAxis.INTERACTIONS:
        pvals = pvals.T.apply(fdr).T
    else:
        raise NotImplementedError(f"FDR correction for `{corr_axis}` is not implemented.")
    return pvals


def _normalise_interactions(interactions: Any) -> pd.DataFrame:
    """Upper-case gene symbols, drop missing / repeated interactions (``_ligrec.py:203-218``)."""
    inter = _as_interaction_frame(interactions)
    inter[SOURCE] = inter[SOURCE].str.upper()
    inter[TARGET] = inter[TARGET].str.upper()
    return inter.dropna(subset=[SOURCE, TARGET], how="any").drop_duplicates(subset=[SOURCE, TARGET], keep="first")


def _filter_interactions(inter: pd.DataFrame, columns: pd.Index) -> tuple[pd.DataFrame, list]:
    """The interactions whose genes are both among ``columns``, and the genes of the test in its column order."""
    inter = inter[inter[SOURCE].isin(columns) & inter[TARGET].isin(columns)]
    if inter.empty:
        raise ValueError("After filtering by genes, no interactions remain.")
    genes = list(set(inter[SOURCE]) | set(inter[TARGET]))
    return inter.drop_duplicates(subset=[SOURCE, TARGET], keep="first"), genes


def _cluster_pairs(clusters: Any, cats: pd.Index, known: pd.Index) -> list:
    """The sorted (cluster_1, cluster_2) pairs of the test: every pair of ``cats`` by default, a list of names means all their
    pairs; every name must be one of ``known``."""
    if clusters is None:
        clusters = list(map(str, cats))
    if all(isinstance(c, str) for c in clusters):
        clusters = list(product(clusters, repeat=2))
    checked = []
    for needle in clusters:
        if len(needle) != 2:
            raise ValueError(f"Expected a `tuple` of length `2`, found `{len(needle)}`.")
        for c in needle:
            if c not in known:
                raise ValueError(f"Invalid cluster `{c!r}`.")
        checked.append(tuple(needle))
    return sorted(checked)


class _Selection(NamedTuple):
    """What ``ligrec`` tests, built from var names and obs alone: the host path's ``sub`` frame is ``X[rows][:, gene_pos]``
    (NaN -> 0) with columns ``0 .. len(gene_pos) - 1`` and clusters ``codes``."""

    gene_pos: np.ndarray  # int64 column of X of every gene of the test, in the test's gene order
    rows: np.ndarray  # int64 ascending cells of the selected clusters
    codes: np.ndarray  # int32 cluster code of every selected cell, in [0, n_cls)
    n_cls: int
    inter_: np.ndarray  # (n_interactions, 2) gene indices of the test
    clusters_: np.ndarray  # (n_cluster_pairs, 2) cluster codes
    clusters: list  # sorted (cluster_1, cluster_2) names
    pairs: pd.DataFrame  # (source, target) of every interaction
    inter: pd.DataFrame  # the filtered interactions (metadata columns)


class _ComplexColumns:
    """Stands in for the host path's gene frame in ``_resolve_complexes``: its column names, and the values of the complex
    components that ``complex_policy='min'`` averages (read once, for every component at a time)."""

    def __init__(self, columns: pd.Index, frame: pd.DataFrame):
        self.columns = columns
        self._frame = frame

    def __getitem__(self, parts):
        return self._frame[parts]


def _select_by_names(adata: Any, var_names: Any, cluster_key: str, interactions: Any, complex_policy: str, n_perms: int, clusters: Any,
                     read_columns) -> _Selection:
    """The gene, cell and cluster selection of ``ligrec`` without the expression matrix, step for step as the host path builds
    it from the dense frame.  ``read_columns(positions)`` returns ``X[:, positions]`` over every cell with NaN written as 0 in
    X's own dtype; it is called once, only under ``complex_policy='min'`` and only for complex components."""
    complex_policy = ComplexPolicy(complex_policy)
    inter = _normalise_interactions(interactions)
    # upper-cased gene symbols, repeated ones dropped (the first is kept)
    upper = pd.Index(var_names).astype(str).str.upper()
    keep = ~upper.duplicated()
    columns, col_pos = upper[keep], np.flatnonzero(keep)
    position = dict(zip(columns, col_pos, strict=True))
    parts: dict = {}
    if complex_policy == ComplexPolicy.MIN:
        for name in pd.concat([inter[SOURCE], inter[TARGET]]):
            if isinstance(name, str) and "_" in name:
                parts.update((c, None) for c in name.split("_") if c in position)
    if parts:
        part_index = columns[np.isin(columns, list(parts))]
        frame = pd.DataFrame(read_columns(np.array([position[c] for c in part_index], dtype=np.int64)), columns=part_index)
    else:
        frame = pd.DataFrame(columns=columns[:0])
    inter = _resolve_complexes(inter, _ComplexColumns(columns, frame), complex_policy)
    inter, genes = _filter_interactions(inter, columns)

    # ---- test (PermutationTest.test, :230-370)
    assert_positive(n_perms, name="n_perms")
    assert_categorical_obs(adata, key=cluster_key)
    cats = adata.obs[cluster_key].cat.categories
    if len(cats) <= 1:
        raise ValueError(f"Expected at least `2` clusters, found `{len(cats)}`.")
    pairs_df = inter[[SOURCE, TARGET]]
    labels = pd.Series(adata.obs[cluster_key].astype("string").astype("category").values)
    clusters = _cluster_pairs(clusters, cats, labels.cat.categories)
    flat = list({c for cs in clusters for c in cs})
    rows = np.flatnonzero(np.isin(labels, flat))
    cat = labels.iloc[rows].cat.remove_unused_categories().cat
    cluster_mapper = dict(zip(cat.categories, range(len(cat.categories)), strict=False))
    gene_mapper = dict(zip(genes, range(len(genes)), strict=False))
    clusters_ = np.array([[cluster_mapper[a], cluster_mapper[b]] for a, b in clusters], dtype=np.uint32)
    inter_ = np.vectorize(lambda g: gene_mapper[g])(pairs_df.values)
    return _Selection(np.array([position[g] for g in genes], dtype=np.int64), rows.astype(np.int64), np.asarray(cat.codes, dtype=np.int32),
                      len(cat.categories), inter_, clusters_, clusters, pairs_df, inter)


def ligrec(adata: Any, cluster_key: str, interactions: Any = None, complex_policy: str = ComplexPolicy.MIN.v, threshold: float = 0.01,
           corr_method: str | None = None, corr_axis: str = CorrAxis.CLUSTERS.v, use_raw: bool = True, copy: bool = False,
           key_added: str | None = None, gene_symbols: str | None = None, *, n_perms: int = 1000, seed: int | None = None,
           clusters: Any = None, alpha: float = 0.05, n_jobs: int | None = None, show_progress_bar: bool = True,
           table_key: str | None = None, device: int | None = None) -> Mapping[str, pd.DataFrame] | None:
    """Permutation test of receptor-ligand interactions between clusters (``_ligrec.py:543-613``); returns / writes
    ``adata.uns[f'{cluster_key}_ligrec'] = {'means', 'pvalues', 'metadata'}`` (frames indexed by (source, target), columns
    (cluster_1, cluster_2)).  ``n_jobs`` / ``show_progress_bar`` are accepted and ignored.
    Under an initialised ``torch.distributed`` process group (one process per GPU) the permutations are sharded over the ranks
    and the permutation counts summed once over them; every rank gets the full result."""
    adata = extract_adata_if_sdata(adata, table_key=table_key)
    if not adata.shape[0]:
        raise ValueError("No cells are in `adata.obs_names`.")
    if not adata.shape[1]:
        raise ValueError("No genes are in `adata.var_names`.")
    src_adata = adata
    if use_raw:
        if adata.raw is None:
            raise AttributeError("No `.raw` attribute found. Try specifying `use_raw=False`.")
        src_adata = adata.raw
    var_names = src_adata.var_names if gene_symbols is None else src_adata.var[gene_symbols]
    if device_matrix(src_adata.X) is not None:
        m, ctx = device_context(src_adata.X, device)
        if m.shape[0] != adata.shape[0]:
            raise ValueError(f"Expected the expression matrix to have `{adata.shape[0]}` rows, found `{m.shape[0]}`.")

        def read_columns(positions):  # X[:, positions] over every cell, NaN -> 0, in X's own dtype (pandas' fillna(0.0) frame)
            with ctx.lock, Gathered(ctx, m, None, positions, OBS_MAJOR, nan_zero=True, keep_dtype=True) as g:
                return g.download()

        sel = _select_by_names(adata, var_names, cluster_key, interactions, complex_policy, n_perms, clusters, read_columns)
        pairs_df, clusters, inter = sel.pairs, sel.clusters, sel.inter
        if corr_method is not None:
            corr_axis = CorrAxis(corr_axis)
        start = time.perf_counter()
        logg.info("Running `%d` permutations on `%d` interactions and `%d` cluster combinations on the GPU", n_perms, len(pairs_df), len(clusters))
        with ctx.lock, Gathered(ctx, m, sel.rows, sel.gene_pos, OBS_MAJOR, nan_zero=True) as x:
            res_t = ligrec_analysis_device(x, sel.codes, sel.n_cls, sel.inter_, sel.clusters_, threshold=threshold, n_perms=int(n_perms),
                                           seed=seed)
        return _finish(adata, res_t, pairs_df, clusters, inter, corr_method, corr_axis, alpha, copy, cluster_key, key_added, start)
    from scipy.sparse import issparse

    X = src_adata.X
    X = X.toarray() if issparse(X) else np.asarray(X)
    data = pd.DataFrame(X, index=adata.obs_names, columns=pd.Index(var_names).astype(str)).fillna(0.0)

    complex_policy = ComplexPolicy(complex_policy)
    inter = _normalise_interactions(interactions)
    # upper-cased gene symbols, repeated ones dropped (the first is kept)
    data.columns = data.columns.str.upper()
    data = data.loc[:, ~data.columns.duplicated()]
    inter = _resolve_complexes(inter, data, complex_policy)
    inter, genes = _filter_interactions(inter, data.columns)
    filtered = data.loc[:, genes].copy()

    # ---- test (PermutationTest.test, :230-370)
    assert_positive(n_perms, name="n_perms")
    assert_categorical_obs(adata, key=cluster_key)
    if corr_method is not None:
        corr_axis = CorrAxis(corr_axis)
    cats = adata.obs[cluster_key].cat.categories
    if len(cats) <= 1:
        raise ValueError(f"Expected at least `2` clusters, found `{len(cats)}`.")
    pairs_df = inter[[SOURCE, TARGET]]
    filtered["clusters"] = adata.obs[cluster_key].astype("string").astype("category").values
    clusters = _cluster_pairs(clusters, cats, filtered["clusters"].cat.categories)
    flat = list({c for cs in clusters for c in cs})
    sub = filtered.loc[np.isin(filtered["clusters"], flat), :].copy()
    sub["clusters"] = sub["clusters"].cat.remove_unused_categories()
    cat = sub["clusters"].cat
    cluster_mapper = dict(zip(cat.categories, range(len(cat.categories)), strict=False))
    gene_mapper = dict(zip(sub.columns[:-1], range(len(sub.columns) - 1), strict=False))
    sub.columns = [gene_mapper[c] if c != "clusters" else c for c in sub.columns]
    clusters_ = np.array([[cluster_mapper[a], cluster_mapper[b]] for a, b in clusters], dtype=np.uint32)
    sub["clusters"] = cat.rename_categories(cluster_mapper)
    inter_ = np.vectorize(lambda g: gene_mapper[g])(pairs_df.values)

    start = time.perf_counter()
    logg.info("Running `%d` permutations on `%d` interactions and `%d` cluster combinations on the GPU", n_perms, len(pairs_df), len(clusters))
    res_t = ligrec_analysis(sub, inter_, clusters_, threshold=threshold, n_perms=int(n_perms), seed=seed, ctx=default_context(device))
    return _finish(adata, res_t, pairs_df, clusters, inter, corr_method, corr_axis, alpha, copy, cluster_key, key_added, start)


def _finish(adata: Any, res_t: TempResult, pairs_df: pd.DataFrame, clusters: list, inter: pd.DataFrame, corr_method: str | None, corr_axis: Any,
            alpha: float, copy: bool, cluster_key: str, key_added: str | None, start: float) -> Mapping[str, pd.DataFrame] | None:
    """The result frames (``PermutationTest.test``, ``_ligrec.py:330-370``), returned or written to ``adata.uns``."""
    index = pd.MultiIndex.from_frame(pairs_df, names=[SOURCE, TARGET])
    columns = pd.MultiIndex.from_tuples(clusters, names=["cluster_1", "cluster_2"])
    res: dict[str, pd.DataFrame] = {
        "means": pd.DataFrame({c: pd.arrays.SparseArray(res_t.means[:, i], fill_value=0) for i, c in enumerate(columns)}, index=index),
        "pvalues": pd.DataFrame({c: pd.arrays.SparseArray(res_t.pvalues[:, i], fill_value=np.nan) for i, c in enumerate(columns)}, index=index),
        "metadata": inter[inter.columns.difference([SOURCE, TARGET])],
    }
    res["metadata"].index = res["means"].index.copy()
    if corr_method is not None:
        res["pvalues"] = _fdr_correct(res["pvalues"], corr_method, corr_axis, alpha)
    if copy:
        logg.info("Finish (%.3fs)", time.perf_counter() - start)
        return res
    _save_data(adata, attr="uns", key=Key.uns.ligrec(cluster_key, key_added), data=res, time_start=start)
    return None
