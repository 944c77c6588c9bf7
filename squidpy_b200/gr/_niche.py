"""Niche calling: ``calculate_niche`` and its flavours (``src/squidpy/gr/_niche.py``), with the embeddings on the GPU.

The embedding each flavour clusters is built on the device (``csrc/niche.cu``): neighbourhood profiles over 1..``distance``
hops, UTAG's ``normalize(A, "l1") @ X`` and CellCharter's hop aggregates.  What follows the embedding is the reference's
own: scanpy's ``pp.scale`` / ``tl.pca`` / ``pp.neighbors`` / ``tl.leiden`` and scikit-learn's ``GaussianMixture``, called
with the same arguments on the same temporary AnnData contents.  scanpy is imported when a flavour needs it; without it
those flavours raise ``ImportError`` before any GPU work.  ``flavor="spatialleiden"`` has no embedding step and is not
provided.
"""

from __future__ import annotations

import warnings
from typing import Any

import numpy as np
import pandas as pd

from .._adata import AnnDataLite
from .._device import DevArray, DevSparse, array_device, device_matrix, graph_value_code, matrix_args
from .._lib import check, default_context, load, pointer_device
from .._validators import assert_key_in_adata, extract_adata_if_sdata
from ._utils import caller_graph, logg

__all__ = ["calculate_niche", "calculate_niche_neighborhood", "calculate_niche_utag", "calculate_niche_cellcharter", "niche_profile",
           "niche_aggregate"]

NOT_A_NICHE = "not_a_niche"
_FLAVORS = ["neighborhood", "utag", "cellcharter", "spatialleiden"]


# ---------------------------------------------------------------------------------------------------------------------
# Device calls
# ---------------------------------------------------------------------------------------------------------------------
# scipy multiplies and adds boolean matrices as logical and / or: the reference's A^k of a boolean graph is reachability and its
# hop comparison True > True is False.  The embeddings here are path sums, so a boolean graph would give other numbers.
_BOOL_GRAPH = ("Boolean connectivity graphs are not supported: scipy combines their entries with logical and / or, which the niche "
               "embeddings do not reproduce.  Pass the graph with numeric values, e.g. `A.astype(np.float32)`.")


def _graph_abi(conn: Any, n: int, device: int | None) -> tuple[tuple, int | None, bool]:
    """``(graph arguments of sqb_niche_*, device, float32 values)`` of a host or device neighbour graph."""
    g = caller_graph(conn, n, device)
    if g.dev is None:
        if g.host.dtype == np.float32 or g.host.dtype == np.float64:
            data, code = np.ascontiguousarray(g.host.data), 0 if g.host.dtype == np.float32 else 1
        elif g.host.dtype == np.bool_:
            raise TypeError(_BOOL_GRAPH)
        elif g.host.dtype.kind in "iu":
            data, code = np.ascontiguousarray(g.host.data, dtype=np.int64), 4
        else:
            raise TypeError(f"Graph values of dtype `{g.host.dtype}` are not supported.")
        data_ptr = data.ctypes.data
    else:
        code = graph_value_code(g.dev.data, g.index_args[1])
        if code == 5:
            raise TypeError(_BOOL_GRAPH)
        if code == 2:
            raise TypeError("Device graph values of dtype `float16` are not supported; use float32, float64, int32 or int64.")
        data = g.dev.data
        data_ptr = data.ptr or None
    args = (*g.index_args, data_ptr, code, int(g.csc), int(g.dev is not None), g.stream)
    return (args, (g, data)), g.device, code == 0


def niche_profile(conn: Any, codes: np.ndarray, n_cls: int, distance: int = 1, weights: list[float] | None = None,
                  abs_nhood: bool = False, *, device: int | None = None) -> np.ndarray:
    """The neighbourhood-profile embedding (``sqb_niche_profile``): float64 ``n x n_cls``.  ``codes``: int32 category codes,
    -1 for NaN.  ``weights``: the hop weights when ``distance > 1`` (extended with their last value when shorter, their full sum
    divides the result unless ``abs_nhood``)."""
    codes = np.ascontiguousarray(codes, dtype=np.int32)
    n = codes.size
    distance = max(int(distance), 1)
    (args, keep), device, _ = _graph_abi(conn, n, device)
    if distance > 1:
        w = [1.0] * distance if weights is None else list(weights)
        if len(w) < distance:
            w = w + [w[-1]] * (distance - len(w))
        wsum = float(sum(w))
        w_arr = np.ascontiguousarray(w[:distance], dtype=np.float64)
    else:
        wsum, w_arr = 1.0, None
    out = np.empty((n, n_cls), dtype=np.float64)
    if n_cls == 0:
        return out
    ctx = default_context(device)
    with ctx.lock:
        check(load().sqb_niche_profile(ctx.handle, *args, codes.ctypes.data, int(n_cls), distance,
                                       None if w_arr is None else w_arr.ctypes.data, wsum, int(bool(abs_nhood)), out.ctypes.data))
    del keep
    return out


def _x_abi(X: Any, n: int, f32: bool) -> tuple[tuple, Any, int | None]:
    """``(X arguments of sqb_niche_aggregate, owner, device)``: a host or device matrix, dense or CSR, in float32 / float64."""
    import scipy.sparse as sp

    dtype = np.float32 if f32 else np.float64
    d = device_matrix(X)
    if d is None:
        if sp.issparse(X):
            csr = X.tocsr() if X.format != "csr" else X
            if csr.shape[0] != n:
                raise ValueError(f"Expected `X` with `{n}` rows, found `{csr.shape[0]}`.")
            ip, ix = (np.ascontiguousarray(a) if a.dtype in (np.int32, np.int64) else np.ascontiguousarray(a, np.int64)
                      for a in (csr.indptr, csr.indices))
            v = np.ascontiguousarray(csr.data, dtype=dtype)
            return ((v.ctypes.data, ip.ctypes.data, ix.ctypes.data, ix.size, 1, 8 * ip.itemsize, 8 * ix.itemsize, int(f32), csr.shape[1], 0, 0),
                    (v, ip, ix), None)
        a = np.ascontiguousarray(np.asarray(X), dtype=dtype)
        if a.ndim != 2 or a.shape[0] != n:
            raise ValueError(f"Expected a 2-D `X` with `{n}` rows, found shape `{a.shape}`.")
        return (a.ctypes.data, None, None, 0, 0, 32, 32, int(f32), a.shape[1], 0, 0), a, None
    import torch  # a device matrix in another layout or dtype is rearranged by torch on its own device

    if isinstance(X, torch.Tensor):
        tdt = torch.float32 if f32 else torch.float64
        if X.layout == torch.strided:
            X = X.to(tdt).contiguous()
        elif X.layout == torch.sparse_csc or X.dtype != tdt:
            X = X.to_sparse_csr().to(tdt) if X.layout != torch.sparse_csr else X.to(tdt)
        d = device_matrix(X)
    m = matrix_args(d, (n, int(d.shape[1])))
    if m.dtype != np.dtype(dtype) or m.format == 2 or (m.format == 0 and m.strides != (m.shape[1], 1)):
        raise TypeError(f"A device `X` must be a C-contiguous dense or CSR matrix of `{np.dtype(dtype)}` here, found `{m.dtype}`.")
    on = array_device(d, pointer_device)
    return ((m.x or None, m.indptr or None, m.indices or None, m.nnz, m.format, m.indptr_bits, m.index_bits, int(f32), m.shape[1], 1, m.stream),
            X, on)


def _x_dtype(X: Any) -> np.dtype:
    d = device_matrix(X)
    if d is None:
        return np.dtype(X.dtype)
    return np.dtype((d.data if isinstance(d, DevSparse) else d).dtype)


def niche_aggregate(conn: Any, X: Any, mode: str, distance: int = 1, *, device: int | None = None) -> tuple[np.ndarray, np.ndarray]:
    """``sqb_niche_aggregate``: ``mode="utag"`` gives ``normalize(A, "l1") @ X``; ``"mean"`` / ``"variance"`` give CellCharter's
    dense ``[X, agg_1, ..., agg_distance]``.  Returns ``(out, hop_nnz)`` with the output in the dtype scipy's upcast gives."""
    n = int(X.shape[0])
    (gargs, gkeep), gdev, w_f32 = _graph_abi(conn, n, device)
    x_dt = _x_dtype(X)
    f32 = np.result_type(x_dt, np.float32) == np.float32
    t1 = np.float32 if (w_f32 and f32) else np.float64
    if mode == "utag":
        code, out_dt = 0, np.dtype(t1)
    elif mode in ("mean", "variance"):
        if distance < 1:
            raise ValueError(f"'distance' must be at least 1, got {distance}")
        code = 1 if mode == "mean" else 2
        out_dt = np.result_type(x_dt, t1, *([np.float64] if distance > 1 else []))
    else:
        raise ValueError(f"Invalid aggregation method '{mode}'. Please choose either 'mean' or 'variance'.")
    if out_dt not in (np.float32, np.float64):
        raise TypeError(f"`X` of dtype `{x_dt}` is not supported.")
    xargs, xkeep, xdev = _x_abi(X, n, bool(f32))
    if gdev is not None and xdev is not None and gdev != xdev:
        raise ValueError(f"The connectivity graph (cuda:{gdev}) and `X` (cuda:{xdev}) live on different devices.")
    device = gdev if gdev is not None else xdev if xdev is not None else device
    m = int(xargs[8])
    cols = m if code == 0 else (distance + 1) * m
    out = np.empty((n, cols), dtype=out_dt)
    hop_nnz = np.zeros(max(distance, 1), dtype=np.int64)
    ctx = default_context(device)
    with ctx.lock:
        check(load().sqb_niche_aggregate(ctx.handle, *gargs, *xargs, code, int(distance), int(out_dt == np.float32), out.ctypes.data,
                                         hop_nnz.ctypes.data))
    del gkeep, xkeep
    return out, hop_nnz


# ---------------------------------------------------------------------------------------------------------------------
# The scanpy seam
# ---------------------------------------------------------------------------------------------------------------------
def _scanpy():
    try:
        import scanpy as sc
    except ImportError as e:
        raise ImportError("This niche flavour clusters or reduces the embedding with scanpy: `pip install scanpy`.") from e
    return sc


def _anndata(**kw):
    try:
        from anndata import AnnData
    except ImportError:
        AnnData = AnnDataLite
    return AnnData(**kw)


def _dense(X: Any) -> bool:
    return isinstance(X, np.ndarray) or isinstance(device_matrix(X), DevArray)


def _is_sdata(data: Any) -> bool:
    return getattr(data, "tables", None) is not None and not hasattr(data, "obsp")


# ---------------------------------------------------------------------------------------------------------------------
# Embedders and clusterers
# ---------------------------------------------------------------------------------------------------------------------
class _Profile:
    def __init__(self, groups, key, scale, distance, abs_nhood, n_hop_weights, device):
        self.groups, self.key, self.scale, self.distance = groups, key, scale, distance
        self.abs_nhood, self.n_hop_weights, self.device = abs_nhood, n_hop_weights, device

    def embed(self, adata: Any) -> np.ndarray:
        col = adata.obs[self.groups]
        if col.dtype.name != "category":
            warnings.warn("Since adata.obs[groups] does not already have categorical dtype, converting it into categorical type.", stacklevel=3)
            adata.obs[self.groups] = col = col.astype("category")
        codes = np.asarray(col.cat.codes, dtype=np.int32)
        prof = niche_profile(adata.obsp[self.key], codes, len(col.cat.categories), self.distance if self.distance > 1 else 1,
                             self.n_hop_weights, self.abs_nhood, device=self.device)
        emb = _anndata(X=prof, obs=pd.DataFrame(index=col.index))
        if self.scale:
            _scanpy().pp.scale(emb, zero_center=True)
        return emb.X


class _Utag:
    def __init__(self, key, device):
        self.key, self.device = key, device

    def embed(self, adata: Any) -> np.ndarray:
        import scipy.sparse as sp

        out, _ = niche_aggregate(adata.obsp[self.key], adata.X, "utag", device=self.device)
        # a sparse X gives a sparse product in the reference, and scanpy's PCA treats the two differently
        emb = _anndata(X=out if _dense(adata.X) else sp.csr_matrix(out))
        _scanpy().tl.pca(emb)
        return emb.obsm["X_pca"]


class _CellCharter:
    def __init__(self, distance, aggregation, key, n_components, use_rep, device):
        self.distance, self.aggregation, self.key = distance, aggregation, key
        self.n_components, self.use_rep, self.device = n_components, use_rep, device

    def embed(self, adata: Any) -> np.ndarray:
        if self.use_rep is not None:
            assert_key_in_adata(adata, self.use_rep, attr="obsm")
            rep = adata.obsm[self.use_rep]
            if rep.shape[1] < self.n_components:
                raise ValueError(
                    f"Embedding has {rep.shape[1]} components, but n_components={self.n_components}. Please provide an embedding with at "
                    f"least {self.n_components} components."
                )
            return rep[:, : self.n_components]
        logg.warning(
            "CellCharter recommends to use a dimensionality reduced embedding of the data, e.g. a scVI embedding. Since 'use_rep' is not "
            "provided, PCA will be used as proxy - performance may be suboptimal."
        )
        if self.aggregation not in ("mean", "variance"):
            raise ValueError(f"Invalid aggregation method '{self.aggregation}'. Please choose either 'mean' or 'variance'.")
        if _dense(adata.X):
            # the reference fails on a dense X: the variance densifies the mean with `.toarray()`, which a dense product does not
            # have, and scipy's hstack of the mean's all-dense blocks refuses them
            if self.aggregation == "variance":
                raise AttributeError("'numpy.ndarray' object has no attribute 'toarray'")
            raise ValueError("blocks must be 2-D, and some must be sparse")
        arr, _ = niche_aggregate(adata.obsp[self.key], adata.X, self.aggregation, self.distance, device=self.device)
        emb = _anndata(X=arr)
        _scanpy().tl.pca(emb)
        return emb.obsm["X_pca"]


class _Leiden:
    def __init__(self, n_neighbors, resolutions, base):
        self.n_neighbors, self.base = n_neighbors, base
        self.resolutions = resolutions if isinstance(resolutions, list) else [resolutions]

    def cluster(self, adata: Any, embedding: Any) -> list[str]:
        sc = _scanpy()
        emb = _anndata(X=embedding, obs=pd.DataFrame(index=adata.obs.index))
        sc.pp.neighbors(emb, n_neighbors=self.n_neighbors, use_rep="X")
        keys = []
        for res in self.resolutions:
            key = f"{self.base}_res={res}"
            keys.append(key)
            if key in adata.obs.columns:
                logg.info(f"Overwriting existing column '{key}'")
            sc.tl.leiden(emb, resolution=res, key_added=key)
            adata.obs[key] = list(emb.obs[key])
        return keys


class _GMM:
    def __init__(self, n_components, random_state, base):
        self.n_components, self.random_state, self.base = n_components, random_state, base

    def cluster(self, adata: Any, embedding: Any) -> list[str]:
        from sklearn.mixture import GaussianMixture

        gmm = GaussianMixture(n_components=self.n_components, random_state=self.random_state, init_params="random_from_data")
        gmm.fit(embedding)
        labels = gmm.predict(embedding)
        if self.base in adata.obs.columns:
            logg.info(f"Overwriting existing column '{self.base}'")
        adata.obs[self.base] = pd.Categorical(labels)
        return [self.base]


# ---------------------------------------------------------------------------------------------------------------------
# Pipeline
# ---------------------------------------------------------------------------------------------------------------------
def _postprocess_niche_results(adata: Any, result_columns: list[str], mask: pd.Series | None = None, min_niche_size: int | None = None,
                               prefix: str | None = None) -> None:
    """Relabel the niche columns in place: ``mask`` False -> ``"not_a_niche"``, niches smaller than ``min_niche_size`` ->
    ``"not_a_niche"``, then ``prefix`` before every label.  Labels become strings when any option is given."""
    if mask is None and min_niche_size is None and prefix is None:
        return
    for col in result_columns:
        labels = adata.obs[col].astype(str)
        if mask is not None:
            inside = mask[mask.index.isin(adata.obs.index)]
            labels[~inside] = NOT_A_NICHE
        if min_niche_size is not None:
            sizes = labels.value_counts()
            labels[labels.isin(sizes.index[sizes < min_niche_size])] = NOT_A_NICHE
        if prefix is not None:
            labels = prefix + labels
        adata.obs[col] = labels


def _run_niche_pipeline(adata, embedder, clusterer, mask, min_niche_size, prefix=None) -> None:
    columns = clusterer.cluster(adata, embedder.embed(adata))
    _postprocess_niche_results(adata, columns, mask, min_niche_size, prefix)


def _calculate_niche_custom(data, embedder, clusterer, min_niche_size=None, mask=None, library_key=None, inplace=True, table_key=None):
    """Embed, cluster and relabel ``data`` (a copy unless ``inplace``), library by library when ``library_key`` is given: each
    library runs on ``adata[lib_indices].copy()``, its labels get the prefix ``lib={id}_`` and other rows ``"not_a_niche"``."""
    orig = extract_adata_if_sdata(data, table_key=table_key)
    adata = orig if inplace else orig.copy()
    if library_key is None:
        _run_niche_pipeline(adata, embedder, clusterer, mask, min_niche_size)
    else:
        assert_key_in_adata(adata, library_key, attr="obs")
        logg.info(f"Stratifying by library_key '{library_key}'")
        added: list[str] = []
        for i, lib in enumerate(adata.obs[library_key].unique()):
            logg.info(f"Processing library '{lib}'")
            inside = (adata.obs[library_key] == lib).to_numpy()
            rows = adata.obs.index[inside]
            if len(rows) == 0:
                logg.warning(f"Library '{lib}' contains no cells, skipping")
                continue
            part = adata[inside].copy()  # by position: obs names may repeat or be integers
            _run_niche_pipeline(part, embedder, clusterer, mask, min_niche_size, prefix=f"lib={lib}_")
            if i == 0:
                added = list(set(part.obs.columns) - set(adata.obs.columns))
            for col in added:
                if col not in adata.obs:
                    adata.obs[col] = NOT_A_NICHE
                adata.obs.loc[rows, col] = list(part.obs[col].astype("str"))
    if _is_sdata(data):
        from spatialdata import sanitize_table

        sanitize_table(adata)
    return None if inplace else adata


# ---------------------------------------------------------------------------------------------------------------------
# Validation (calculate_niche)
# ---------------------------------------------------------------------------------------------------------------------
def _assert_isinstance(value: Any, types: type | tuple[type, ...], name: str) -> None:
    if not isinstance(value, types):
        names = " or ".join(t.__name__ for t in types) if isinstance(types, tuple) else types.__name__
        raise TypeError(f"Expected `{name}` to be of type `{names}`, got `{type(value).__name__}`.")


def _assert_one_of(value: Any, options: list, name: str) -> None:
    if value not in options:
        raise ValueError(f"Expected `{name}` to be one of `{list(options)}`, got `{value!r}`.")


# per flavour: the arguments that must not be None, and those it ignores (a value other than the default is reported)
_REQUIRED = {
    "neighborhood": ["groups", "n_neighbors", "resolutions", "spatial_connectivities_key"],
    "utag": ["n_neighbors", "resolutions", "spatial_connectivities_key"],
    "cellcharter": ["distance", "aggregation", "random_state", "spatial_connectivities_key"],
    "spatialleiden": ["latent_connectivities_key", "spatial_connectivities_key"],
}
_UNUSED = {
    "neighborhood": ["aggregation", "n_components", "random_state", "latent_connectivities_key", "layer_ratio", "n_iterations", "use_weights",
                     "use_rep"],
    "utag": ["groups", "min_niche_size", "scale", "abs_nhood", "distance", "n_hop_weights", "aggregation", "n_components", "random_state",
             "latent_connectivities_key", "layer_ratio", "n_iterations", "use_weights", "use_rep"],
    "cellcharter": ["groups", "min_niche_size", "scale", "abs_nhood", "n_neighbors", "resolutions", "n_hop_weights", "latent_connectivities_key",
                    "layer_ratio", "n_iterations", "use_weights"],
    "spatialleiden": ["groups", "min_niche_size", "scale", "abs_nhood", "n_neighbors", "n_hop_weights", "use_rep"],
}
_CHECKED_UNUSED = ("groups", "n_neighbors", "resolutions", "min_niche_size", "scale", "abs_nhood", "distance", "n_hop_weights", "aggregation",
                   "n_components", "random_state", "use_rep")
_DEFAULTS = {"scale": True, "abs_nhood": False, "random_state": 42}


def _check_unnecessary_args(flavor: str, values: dict[str, Any], unused: list[str]) -> None:
    """Warn (through the logger) about the arguments ``flavor`` ignores that were given a value other than their default."""
    given = []
    for name in unused:
        v = values.get(name)
        if name in _DEFAULTS and (v == _DEFAULTS[name] if name == "random_state" else v is _DEFAULTS[name]):
            continue
        if v is not None:
            given.append(name)
    if given:
        logg.warning(f"Parameters {', '.join(given)} are not used for flavor '{flavor}'.")


def _validate_niche_args(data, flavor, library_key, table_key, groups, n_neighbors, resolutions, min_niche_size, scale, abs_nhood, distance,
                         n_hop_weights, aggregation, n_components, random_state, spatial_connectivities_key, latent_connectivities_key,
                         layer_ratio, n_iterations, use_weights, use_rep, inplace) -> None:
    """The reference's argument checks for ``calculate_niche``: same exception types, messages and order."""
    if not (hasattr(data, "obs") and hasattr(data, "obsp")) and not _is_sdata(data):
        raise TypeError(f"Expected `data` to be of type `AnnData or SpatialData`, got `{type(data).__name__}`.")
    _assert_one_of(flavor, _FLAVORS, "flavor")
    if _is_sdata(data) and table_key is None:
        raise TypeError("missing required keyword-only argument: 'table_key'")
    if library_key is not None:
        _assert_isinstance(library_key, str, "library_key")
        if library_key not in extract_adata_if_sdata(data, table_key=table_key).obs.columns:
            raise ValueError(f"'library_key' must be a column in 'adata.obs', got {library_key}")
    if n_neighbors is not None:
        _assert_isinstance(n_neighbors, int, "n_neighbors")
    if resolutions is not None:
        if not isinstance(resolutions, float | tuple | list):
            raise TypeError("'resolutions' must be a float, a tuple of floats, a list of floats, or a list containing floats and/or tuples of "
                            f"floats, got {type(resolutions).__name__}")
        if isinstance(resolutions, tuple) and not all(isinstance(r, float) for r in resolutions):
            raise TypeError("All elements in the tuple 'resolutions' must be floats.")
        if isinstance(resolutions, list):
            for r in resolutions:
                if not (isinstance(r, float) or (isinstance(r, tuple) and all(isinstance(x, float) for x in r))):
                    raise TypeError("Each item in the list 'resolutions' must be a float or a tuple of floats.")
    if n_hop_weights is not None:
        _assert_isinstance(n_hop_weights, list, "n_hop_weights")
    _assert_isinstance(scale, bool, "scale")
    _assert_isinstance(abs_nhood, bool, "abs_nhood")
    values = dict(groups=groups, n_neighbors=n_neighbors, resolutions=resolutions, min_niche_size=min_niche_size, scale=scale,
                  abs_nhood=abs_nhood, distance=distance, n_hop_weights=n_hop_weights, aggregation=aggregation, n_components=n_components,
                  random_state=random_state, use_rep=use_rep, spatial_connectivities_key=spatial_connectivities_key,
                  latent_connectivities_key=latent_connectivities_key)
    for name in _REQUIRED[flavor]:
        if values[name] is None:
            raise ValueError(f"'{name}' is required for flavor '{flavor}'")
    _check_unnecessary_args(flavor, {k: values[k] for k in _CHECKED_UNUSED}, _UNUSED[flavor])
    if flavor == "neighborhood":
        _assert_isinstance(groups, str, "groups")
        if min_niche_size is not None:
            _assert_isinstance(min_niche_size, int, "min_niche_size")
        if isinstance(distance, int) and distance < 1:
            raise ValueError(f"'distance' must be at least 1, got {distance}")
    elif flavor == "cellcharter":
        if distance is not None:
            _assert_isinstance(distance, int, "distance")
            if distance < 1:
                raise ValueError(f"'distance' must be at least 1, got {distance}")
        if aggregation is not None:
            _assert_isinstance(aggregation, str, "aggregation")
            _assert_one_of(aggregation, ["mean", "variance"], "aggregation")
        _assert_isinstance(n_components, int, "n_components")
        if n_components < 1:
            raise ValueError(f"'n_components' must be at least 1, got {n_components}")
        _assert_isinstance(random_state, int, "random_state")
        if use_rep is not None:
            _assert_isinstance(use_rep, str, "use_rep")
    elif flavor == "spatialleiden":
        _assert_isinstance(latent_connectivities_key, str, "latent_connectivities_key")
        _assert_isinstance(spatial_connectivities_key, str, "spatial_connectivities_key")
        _assert_isinstance(layer_ratio, (float, int), "layer_ratio")
        _assert_isinstance(n_iterations, int, "n_iterations")
        if not (isinstance(use_weights, bool) or (isinstance(use_weights, tuple) and len(use_weights) == 2
                                                  and all(isinstance(x, bool) for x in use_weights))):
            raise TypeError(f"'use_weights' must be a bool or a tuple of two bools, got {use_weights!r}")
        _assert_isinstance(random_state, int, "random_state")
    _assert_isinstance(inplace, bool, "inplace")


# ---------------------------------------------------------------------------------------------------------------------
# Public functions
# ---------------------------------------------------------------------------------------------------------------------
def calculate_niche(data: Any, flavor: str, library_key: str | None = None, mask: pd.Series | None = None, groups: str | None = None,
                    n_neighbors: int | None = None, resolutions: float | list | None = None, min_niche_size: int | None = None,
                    scale: bool = True, abs_nhood: bool = False, distance: int | None = None, n_hop_weights: list[float] | None = None,
                    aggregation: str | None = None, n_components: int | None = None, random_state: int = 42,
                    spatial_connectivities_key: str = "spatial_connectivities", latent_connectivities_key: str = "connectivities",
                    layer_ratio: float = 1.0, n_iterations: int = -1, use_weights: bool | tuple[bool, bool] = True, use_rep: str | None = None,
                    inplace: bool = True, *, table_key: str | None = None, device: int | None = None) -> Any:
    """Niches by ``flavor`` (deprecated in the reference since 1.8.4: use the flavour's own function).  Defaults as the
    reference's: ``distance`` 3 for cellcharter and 1 otherwise, ``aggregation="mean"`` and ``n_components=10`` for
    cellcharter, ``resolutions=[0.5]``.  ``device``: the CUDA device of the embedding (the graph's, when it is in GPU memory)."""
    warnings.warn(
        "Calling `calculate_niche` is deprecated and will be removed in squidpy v1.9.0. Use `calculate_niche_neighborhood`, "
        "`calculate_niche_utag`, `calculate_niche_cellcharter`, or `calculate_niche_spatialleiden` instead.",
        FutureWarning,
        stacklevel=2,
    )
    if flavor == "cellcharter":
        aggregation = "mean" if aggregation is None else aggregation
        n_components = 10 if n_components is None else n_components
    if distance is None:
        distance = 3 if flavor == "cellcharter" else 1
    _validate_niche_args(data, flavor, library_key, table_key, groups, n_neighbors, resolutions, min_niche_size, scale, abs_nhood, distance,
                         n_hop_weights, aggregation, n_components, random_state, spatial_connectivities_key, latent_connectivities_key,
                         layer_ratio, n_iterations, use_weights, use_rep, inplace)
    if resolutions is None:
        resolutions = [0.5]
    common = dict(min_niche_size=min_niche_size, mask=mask, library_key=library_key, inplace=inplace, table_key=table_key, device=device)
    if flavor == "neighborhood":
        return calculate_niche_neighborhood(data, groups, resolutions, n_neighbors, spatial_connectivities_key, scale, distance, abs_nhood,
                                            n_hop_weights, **common)
    if flavor == "utag":
        return calculate_niche_utag(data, resolutions, n_neighbors, spatial_connectivities_key, **common)
    if flavor == "cellcharter":
        return calculate_niche_cellcharter(data, distance, aggregation, random_state, spatial_connectivities_key, n_components, use_rep,
                                           **common)
    return calculate_niche_spatialleiden()


def calculate_niche_spatialleiden(*args: Any, **kwargs: Any) -> Any:
    """Not provided: SpatialLeiden has no embedding step and runs entirely in the ``spatialleiden`` package."""
    raise NotImplementedError("flavor='spatialleiden' is not provided by squidpy_b200: call the `spatialleiden` package "
                              "(`spatialleiden.spatialleiden`) directly.")


def calculate_niche_neighborhood(data: Any, groups: str, resolutions: float | list[float], n_neighbors: int = 15,
                                 spatial_connectivities_key: str = "spatial_connectivities", scale: bool = True, distance: int = 1,
                                 abs_nhood: bool = False, n_hop_weights: list[float] | None = None, min_niche_size: int | None = None,
                                 mask: pd.Series | None = None, library_key: str | None = None, inplace: bool = True,
                                 table_key: str | None = None, *, device: int | None = None) -> Any:
    """Leiden niches of the neighbourhood profile: per observation, the frequency of each ``groups`` category among its
    neighbours over 1..``distance`` hops (weighted by ``n_hop_weights``), z-scored when ``scale``.  Adds
    ``nhood_niche_res={r}`` to ``obs``; returns the copy when ``inplace=False``."""
    _scanpy()
    return _calculate_niche_custom(data, _Profile(groups, spatial_connectivities_key, scale, distance, abs_nhood, n_hop_weights, device),
                                   _Leiden(n_neighbors, resolutions, "nhood_niche"), min_niche_size=min_niche_size, mask=mask,
                                   library_key=library_key, inplace=inplace, table_key=table_key)


def calculate_niche_utag(data: Any, resolutions: float | list[float], n_neighbors: int = 15,
                         spatial_connectivities_key: str = "spatial_connectivities", min_niche_size: int | None = None,
                         mask: pd.Series | None = None, library_key: str | None = None, inplace: bool = True, table_key: str | None = None,
                         *, device: int | None = None) -> Any:
    """Leiden niches of UTAG's embedding, the PCA of ``normalize(A, "l1") @ X``.  Adds ``utag_niche_res={r}`` to ``obs``."""
    _scanpy()
    return _calculate_niche_custom(data, _Utag(spatial_connectivities_key, device), _Leiden(n_neighbors, resolutions, "utag_niche"),
                                   min_niche_size=min_niche_size, mask=mask, library_key=library_key, inplace=inplace, table_key=table_key)


def calculate_niche_cellcharter(data: Any, distance: int = 3, aggregation: str = "mean", random_state: int = 42,
                                spatial_connectivities_key: str = "spatial_connectivities", n_components: int = 10, use_rep: str | None = None,
                                min_niche_size: int | None = None, mask: pd.Series | None = None, library_key: str | None = None,
                                inplace: bool = True, table_key: str | None = None, *, device: int | None = None) -> Any:
    """Gaussian-mixture niches of CellCharter's embedding: the PCA of ``[X, agg_1, ..., agg_distance]``, each ``agg_k`` the mean
    (or variance) of X over the cells first reached at hop k; or the first ``n_components`` columns of ``obsm[use_rep]``.
    Adds ``cellcharter_niche`` to ``obs``."""
    if use_rep is None:
        _scanpy()
    return _calculate_niche_custom(data, _CellCharter(distance, aggregation, spatial_connectivities_key, n_components, use_rep, device),
                                   _GMM(n_components, random_state, "cellcharter_niche"), min_niche_size=min_niche_size, mask=mask,
                                   library_key=library_key, inplace=inplace, table_key=table_key)
