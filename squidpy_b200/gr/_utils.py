"""Write-back helper (``src/squidpy/gr/_utils.py:77-86``) and small host utilities."""

from __future__ import annotations

import logging
import time
from typing import Any

import numpy as np

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
