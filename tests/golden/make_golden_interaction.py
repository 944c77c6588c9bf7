"""Generates tests/golden/interaction.npz: the UNMODIFIED reference ``interaction_matrix`` (its NaN-label masking
``g[mask, :][:, mask]`` and its numba kernel ``_interaction_matrix``, src/squidpy/gr/_nhood.py:349-429), loaded from the
squidpy source tree named by ``$SQUIDPY_REF`` through the stub-import loader ``oracle/_refload.py``.  Only runnable where the
reference tree exists; the output is committed.

    python tests/golden/make_golden_interaction.py

The cases are built to tell an exact, ordered float64 sum from any other: weights that cancel (``±1e16`` next to ``1.0``),
weights spread over 1e-300 .. 1e300 with subnormals and ``-0.0``, NaN and ``±inf``, float32 weights over the whole float32
exponent range; non-canonical CSR rows (duplicates with different values, unsorted columns, explicit zeros, empty rows);
NaN labels on rows and columns, an unused category, one category; and integer graphs: int8, int16, int32, int64 near 2^62
(the int64 sums wrap modulo 2^64, as numba's do), int64 values that float64 cannot hold (2^53 + 1), and bool.

Per case: the CSR arrays, the codes (-1 = NaN label), the number of categories, whether the weighted float sums depend on
the order of the additions (``order_sensitive``), and the reference's output for ``weights`` x ``normalized``.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import pandas as pd
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from squidpy_b200._adata import AnnDataLite  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "interaction.npz")
FLAGS = [(False, False), (True, False), (False, True), (True, True)]  # (weights, normalized)


def _rows(n, lo, hi, rng, empty_every=0):
    """indptr / indices of a random CSR with lo..hi entries per row (duplicates and unsorted columns as drawn)."""
    ptr, idx = [0], []
    for r in range(n):
        k = 0 if empty_every and r % empty_every == 0 else int(rng.integers(lo, hi + 1))
        idx += list(rng.integers(0, n, k))
        ptr.append(len(idx))
    return np.asarray(ptr, np.int32), np.asarray(idx, np.int32)


def _csr(data, indices, indptr, n):
    return sp.csr_matrix((data, indices, indptr), shape=(n, n))  # arrays kept as given: no sorting, no summing


def _codes(n, k, rng, nan_frac=0.0, unused=None):
    c = rng.integers(0, k, n)
    if unused is not None:
        c[c == unused] = (unused + 1) % k
    if nan_frac:
        c[rng.random(n) < nan_frac] = -1
    return c


def cases():
    """(name, scipy CSR, codes, n_categories, order_sensitive)."""
    rng = np.random.default_rng(20261018)
    out = []

    # float64: heavy cancellation, a few large terms against many small ones in every cell
    n = 120
    ptr, idx = _rows(n, 4, 14, rng)
    v = rng.choice(np.array([1e16, -1e16, 1.0, -1.0, 3.0, 0.5, 2.0**-30, 1e15 + 1.0, -7e15]), idx.size)
    out.append(("cancel_f64", _csr(v, idx, ptr, n), _codes(n, 3, rng), 3, True))

    # float64: magnitudes 1e-300 .. 1e300, subnormals, -0.0
    n = 150
    ptr, idx = _rows(n, 3, 12, rng)
    v = rng.choice([-1.0, 1.0], idx.size) * rng.random(idx.size) * 10.0 ** rng.uniform(-300, 300, idx.size)
    special = np.array([5e-324, -5e-324, 2.2e-310, -1.1e-312, -0.0, 0.0, 1e300, -1e300, 1.0, 1e-300])
    pick = rng.random(idx.size) < 0.3
    v[pick] = rng.choice(special, pick.sum())
    out.append(("spread_f64", _csr(v, idx, ptr, n), _codes(n, 4, rng), 4, True))

    # float64: cancelling and spread values with NaN and ±inf in a few rows (cells reached by them are NaN / ±inf)
    n = 100
    ptr, idx = _rows(n, 3, 10, rng)
    v = rng.choice([1e16, -1e16, 1.0, 0.1, -0.3, 1e-200], idx.size)
    for pos, x in zip(rng.choice(idx.size, 6, replace=False), [np.nan, np.inf, -np.inf, np.inf, -np.nan, -np.inf]):
        v[pos] = x
    out.append(("nonfinite_f64", _csr(v, idx, ptr, n), _codes(n, 5, rng), 5, True))

    # only subnormals and signed zeros: exact in any order (every partial sum is a multiple of 2^-1074)
    n = 60
    ptr, idx = _rows(n, 2, 8, rng)
    v = rng.choice(np.array([5e-324, -5e-324, 1e-320, -0.0, 0.0]), idx.size)
    out.append(("subnormal_f64", _csr(v, idx, ptr, n), _codes(n, 3, rng), 3, False))

    # float32: exponents over the whole float32 range, float32 subnormals; summed in float64
    n = 150
    ptr, idx = _rows(n, 3, 12, rng)
    v = (rng.choice([-1.0, 1.0], idx.size) * (1 + rng.random(idx.size)) * 2.0 ** rng.integers(-149, 127, idx.size)).astype(np.float32)
    v[rng.random(idx.size) < 0.05] = np.float32(-0.0)
    out.append(("spread_f32", _csr(v, idx, ptr, n), _codes(n, 4, rng), 4, True))

    # non-canonical rows: duplicates with different values, unsorted columns, explicit zeros, every 5th row empty
    n = 90
    ptr, idx = _rows(n, 6, 20, rng, empty_every=5)
    for r in range(1, n, 3):  # repeat the row's first column at its end
        if ptr[r + 1] > ptr[r]:
            idx[ptr[r + 1] - 1] = idx[ptr[r]]
    v = rng.choice([1e16, -1e16, 1.0, 2.5, -0.75, 0.0], idx.size)
    out.append(("messy_f64", _csr(v, idx, ptr, n), _codes(n, 3, rng), 3, True))

    # NaN labels on rows and columns, and an unused category
    n = 200
    ptr, idx = _rows(n, 2, 9, rng)
    v = rng.choice([1e16, -1e16, 1.0, 3.0, -0.5], idx.size) * rng.choice([1.0, 1.0 + 2.0**-52], idx.size)
    out.append(("nan_labels_f64", _csr(v, idx, ptr, n), _codes(n, 6, rng, nan_frac=0.2, unused=2), 6, True))
    v32 = (rng.standard_normal(idx.size) * 10.0 ** rng.integers(-20, 20, idx.size)).astype(np.float32)
    out.append(("nan_labels_f32", _csr(v32, idx, ptr, n), _codes(n, 5, rng, nan_frac=0.3), 5, True))

    # one category: every labelled entry in one cell
    n = 80
    ptr, idx = _rows(n, 2, 10, rng)
    v = rng.standard_normal(idx.size) * 10.0 ** rng.integers(-8, 17, idx.size)
    out.append(("one_category_f64", _csr(v, idx, ptr, n), _codes(n, 1, rng, nan_frac=0.1), 1, True))

    # integer graphs
    n = 120
    ptr, idx = _rows(n, 2, 12, rng)
    for dt in (np.int8, np.int16, np.int32):
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, idx.size, endpoint=True).astype(dt)
        out.append((f"int_{np.dtype(dt).name}", _csr(v, idx, ptr, n), _codes(n, 4, rng, nan_frac=0.1), 4, False))
    v = (rng.integers(0, 2, idx.size) * 2 - 1) * (2**62 - rng.integers(0, 1000, idx.size))  # wraps modulo 2^64
    out.append(("int64_wrap", _csr(v.astype(np.int64), idx, ptr, n), _codes(n, 3, rng), 3, False))
    v = np.where(rng.random(idx.size) < 0.5, 2**53 + 1, 3).astype(np.int64)  # 2^53 + 1 is no float64
    out.append(("int64_2p53", _csr(v, idx, ptr, n), _codes(n, 3, rng, nan_frac=0.1), 3, False))
    v = rng.random(idx.size) < 0.6
    out.append(("bool", _csr(v, idx, ptr, n), _codes(n, 4, rng, nan_frac=0.1), 4, False))
    return out


def make_adata(graph, codes, n_cls):
    cats = [f"c{i}" for i in range(n_cls)]
    obs = pd.DataFrame({"cluster": pd.Categorical.from_codes(np.asarray(codes), categories=cats)},
                       index=[str(i) for i in range(len(codes))])
    return AnnDataLite(X=np.zeros((len(codes), 1)), obs=obs, var=pd.DataFrame(index=["g0"]), obsp={"spatial_connectivities": graph})


def main():
    import numba
    import scipy

    from oracle import _refload

    nh = _refload.load()["nh"]
    out = {"meta": np.array(f"numpy {np.__version__}; scipy {scipy.__version__}; numba {numba.__version__}; reference squidpy "
                            "interaction_matrix (gr/_nhood.py:349-429)")}
    all_cases = cases()
    for i, (name, g, codes, n_cls, sensitive) in enumerate(all_cases):
        out[f"c{i}_name"], out[f"c{i}_sensitive"] = np.array(name), np.array(sensitive)
        out[f"c{i}_indptr"], out[f"c{i}_indices"], out[f"c{i}_data"] = g.indptr, g.indices, g.data
        out[f"c{i}_codes"], out[f"c{i}_ncls"] = np.asarray(codes, dtype=np.int64), np.array(n_cls)
        for weights, normalized in FLAGS:
            with np.errstate(divide="ignore", invalid="ignore"):
                res = nh.interaction_matrix(make_adata(g, codes, n_cls), "cluster", weights=weights, normalized=normalized, copy=True)
            out[f"c{i}_w{int(weights)}_n{int(normalized)}"] = res
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, ":", len(all_cases), "cases")


if __name__ == "__main__":
    main()
