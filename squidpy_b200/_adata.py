"""Minimal duck-typed stand-in for :class:`anndata.AnnData` (``anndata`` is not installed in this image).

The ``gr`` functions only touch ``.obs[key]`` (pandas categorical), ``.obsp[key]`` (scipy CSR), ``.obsm[key]``,
``.uns``, ``.X``/``.layers``/``.raw``, ``.var``, ``.var_names``, ``.shape`` and ``adata[:, genes]`` — exactly the
AnnData surface the reference uses on this path (``src/squidpy/gr/_utils.py:25-86``,
``src/squidpy/gr/_ppatterns.py:154-194``) — so a real AnnData works unchanged; this class exists for the tests,
the benchmark and users without anndata.
"""

from __future__ import annotations

from typing import Any

import numpy as np
import pandas as pd


class AnnDataLite:
    def __init__(self, X=None, obs: pd.DataFrame | None = None, var: pd.DataFrame | None = None, obsm=None, obsp=None,
                 uns=None, layers=None, raw=None, shape: tuple[int, int] | None = None):
        if X is not None:
            shape = X.shape
        elif shape is None:
            n_obs = len(obs) if obs is not None else 0
            n_var = len(var) if var is not None else 0
            shape = (n_obs, n_var)
        self.X = X
        self._shape = tuple(shape)
        self.obs = obs if obs is not None else pd.DataFrame(index=pd.RangeIndex(self._shape[0]).astype(str))
        self.var = var if var is not None else pd.DataFrame(index=pd.RangeIndex(self._shape[1]).astype(str))
        self.obsm = dict(obsm or {})
        self.obsp = dict(obsp or {})
        self.uns = dict(uns or {})
        self.layers = dict(layers or {})
        self.raw = raw

    @property
    def shape(self) -> tuple[int, int]:
        return self._shape

    @property
    def n_obs(self) -> int:
        return self._shape[0]

    @property
    def n_vars(self) -> int:
        return self._shape[1]

    @property
    def var_names(self) -> pd.Index:
        return self.var.index

    @property
    def obs_names(self) -> pd.Index:
        return self.obs.index

    def copy(self) -> "AnnDataLite":
        import copy as _copy

        def dup(v):
            return v.clone() if hasattr(v, "clone") and not hasattr(v, "copy") else v.copy()  # torch tensors clone

        return AnnDataLite(
            X=None if self.X is None else dup(self.X), obs=self.obs.copy(), var=self.var.copy(),
            obsm={k: dup(v) for k, v in self.obsm.items()}, obsp={k: dup(v) for k, v in self.obsp.items()},
            uns=_copy.deepcopy(self.uns), layers={k: dup(v) for k, v in self.layers.items()}, raw=self.raw,
            shape=self._shape,
        )

    def _var_indexer(self, sel: Any) -> np.ndarray:
        if isinstance(sel, slice):
            return np.arange(self.n_vars)[sel]
        if isinstance(sel, (pd.Series, pd.Index)):
            sel = sel.to_numpy()
        sel = np.asarray(sel)
        if sel.dtype == bool:
            return np.flatnonzero(sel)
        if sel.dtype.kind in "iu":
            return sel.astype(np.int64)
        ix = self.var.index.get_indexer(np.atleast_1d(sel))
        if (ix < 0).any():
            missing = [str(s) for s, i in zip(np.atleast_1d(sel), ix) if i < 0]
            raise KeyError(f"Values {missing} are not valid var names or indices.")
        return ix

    def _obs_indexer(self, sel: Any) -> np.ndarray:
        if isinstance(sel, slice):
            return np.arange(self.n_obs)[sel]
        if isinstance(sel, (pd.Series, pd.Index)):
            sel = sel.to_numpy()
        sel = np.asarray(sel)
        if sel.dtype == bool:
            return np.flatnonzero(sel)
        if sel.dtype.kind in "iu":
            return sel.astype(np.int64)
        ix = self.obs.index.get_indexer(np.atleast_1d(sel))
        if (ix < 0).any():
            missing = [str(s) for s, i in zip(np.atleast_1d(sel), ix) if i < 0]
            raise KeyError(f"Values {missing} are not valid obs names or indices.")
        return ix

    def _obs_subset(self, sel: Any) -> "AnnDataLite":
        """``adata[obs]`` / ``adata[obs, :]``: the rows of X, obs, obsm, layers and an AnnDataLite ``raw``, the rows and columns of
        obsp.  Integer selections are positions, as in AnnData; obs names select by label."""
        ri = self._obs_indexer(sel)
        return AnnDataLite(X=None if self.X is None else _take(self.X, ri), obs=self.obs.iloc[ri], var=self.var,
                           obsm={k: _take(v, ri) for k, v in self.obsm.items()}, obsp={k: _take(v, ri, both=True) for k, v in self.obsp.items()},
                           uns=self.uns, layers={k: _take(v, ri) for k, v in self.layers.items()},
                           raw=self.raw[ri] if isinstance(self.raw, AnnDataLite) else self.raw, shape=(len(ri), self.n_vars))

    def __getitem__(self, index):
        if not isinstance(index, tuple):
            return self._obs_subset(index)
        if len(index) == 2 and isinstance(index[1], slice) and index[1] == slice(None) and not (
                isinstance(index[0], slice) and index[0] == slice(None)):
            return self._obs_subset(index[0])
        if len(index) != 2:
            raise NotImplementedError("AnnDataLite only supports `adata[obs]`, `adata[:, vars]` and `adata[obs, vars]` indexing")
        rows, cols = index
        ci = self._var_indexer(cols)
        ri = slice(None) if (isinstance(rows, slice) and rows == slice(None)) else rows
        X = None if self.X is None else self.X[ri][:, ci]
        layers = {k: v[ri][:, ci] for k, v in self.layers.items()}
        obs = self.obs if isinstance(ri, slice) else self.obs.iloc[ri]
        return AnnDataLite(X=X, obs=obs, var=self.var.iloc[ci], obsm=self.obsm if isinstance(ri, slice) else {},
                           obsp=self.obsp if isinstance(ri, slice) else {}, uns=self.uns, layers=layers,
                           shape=(len(obs), len(ci)))


def _take(a: Any, ri: np.ndarray, both: bool = False) -> Any:
    """Rows ``ri`` of ``a`` (and the same columns when ``both``): numpy, scipy, pandas, or a torch tensor, sparse ones included,
    which stay on their device and keep their layout."""
    if hasattr(a, "iloc"):
        return a.iloc[ri, ri] if both else a.iloc[ri]
    import sys

    torch = sys.modules.get("torch")
    if torch is not None and isinstance(a, torch.Tensor):
        idx = torch.as_tensor(ri, dtype=torch.int64, device=a.device)
        if a.layout == torch.strided:
            out = a.index_select(0, idx)
            return out.index_select(1, idx) if both else out
        layout = a.layout
        out = a.to_sparse_coo().index_select(0, idx)
        if both:
            out = out.index_select(1, idx)
        out = out.coalesce()
        return out.to_sparse_csr() if layout == torch.sparse_csr else out.to_sparse_csc() if layout == torch.sparse_csc else out
    return a[ri][:, ri] if both else a[ri]

