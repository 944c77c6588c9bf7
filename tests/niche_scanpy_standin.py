"""A deterministic, recording stand-in for the four scanpy calls niche calling makes (test only).

``install()`` puts a module named ``scanpy`` into ``sys.modules`` whose ``pp.scale``, ``tl.pca``, ``pp.neighbors`` and
``tl.leiden`` record every matrix handed to them (``CALLS``: ``(name, dense float64 copy of X, details)``) and answer with
outputs that depend only on their input: column sums are ``math.fsum`` (correctly rounded, so no host's SIMD reduction order
enters), everything else elementwise numpy:

* ``pp.scale(adata, zero_center=True)``: ``X <- (X - mean) / std`` per column, population std, a zero std taken as 1;
* ``tl.pca(adata)``: ``obsm["X_pca"]`` = the first ``min(10, n_vars)`` columns of dense X, centred;
* ``pp.neighbors(adata, n_neighbors, use_rep="X")``: records only;
* ``tl.leiden(adata, resolution, key_added)``: ``obs[key_added]`` = str(argmax of the row % (1 + int(10 * resolution))).

The golden generator runs the reference through it and the tests run this library through it, so what each hands to
scanpy is compared bit for bit, and the labels end to end.
"""

from __future__ import annotations

import math
import sys
import types

import numpy as np
import pandas as pd

CALLS: list[tuple[str, np.ndarray, dict]] = []


def _dense(X) -> tuple[np.ndarray, dict]:
    import scipy.sparse as sp

    info = {"sparse": bool(sp.issparse(X)), "dtype": str(X.dtype)}
    return (X.toarray() if sp.issparse(X) else np.array(X)), info


def _col_mean(X: np.ndarray) -> np.ndarray:
    return np.array([math.fsum(c) / X.shape[0] for c in X.T]) if X.shape[0] else np.zeros(X.shape[1])


def _scale(adata, zero_center=True):
    X, info = _dense(adata.X)
    CALLS.append(("scale", X.copy(), {**info, "zero_center": zero_center}))
    X = X.astype(np.float64)
    mean = _col_mean(X)
    std = np.sqrt(_col_mean((X - mean) ** 2))
    std[std == 0] = 1.0
    adata.X = (X - mean) / std


def pca_of(X: np.ndarray) -> np.ndarray:
    """The stand-in's ``X_pca`` of a dense X."""
    Y = X[:, : min(10, X.shape[1])].astype(np.float64)
    return Y - _col_mean(Y)


def _pca(adata):
    X, info = _dense(adata.X)
    CALLS.append(("pca", X.copy(), info))
    adata.obsm["X_pca"] = pca_of(X)


def _neighbors(adata, n_neighbors=15, use_rep=None):
    X, info = _dense(adata.X)
    CALLS.append(("neighbors", X.copy(), {**info, "n_neighbors": n_neighbors, "use_rep": use_rep}))


def _leiden(adata, resolution=1.0, key_added="leiden"):
    X, info = _dense(adata.X)
    CALLS.append(("leiden", X.copy(), {**info, "resolution": resolution, "key_added": key_added}))
    k = 1 + int(10 * resolution)
    labels = (np.argmax(X, axis=1) % k).astype(str) if X.shape[1] else np.zeros(X.shape[0], dtype=int).astype(str)
    adata.obs[key_added] = pd.Categorical(labels)


def install() -> types.ModuleType:
    """Register the stand-in as ``scanpy`` (replacing any real one) and clear ``CALLS``."""
    CALLS.clear()
    sc = types.ModuleType("scanpy")
    sc.pp = types.SimpleNamespace(scale=_scale, neighbors=_neighbors)
    sc.tl = types.SimpleNamespace(pca=_pca, leiden=_leiden)
    sc.__dict__["__standin__"] = True
    sys.modules["scanpy"] = sc
    return sc
