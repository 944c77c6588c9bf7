"""CPU checks of the arithmetic the device graph builders follow (csrc/graph_device.cu) against the host builders, and of how
device coordinates are recognised and parsed:

* the percentile threshold from two order statistics (numpy's 'linear' method, the n diagonal zeros leading the sorted
  distances) equals ``np.percentile`` of the host path's ``dst.data``;
* the cosine restatement (sklearn's row normalisation, scipy's csr_matmat accumulation order) equals
  ``cosine_similarity(adj, dense_output=False)`` bit for bit;
* the level-by-level ring expansion equals ``GridBuilder(n_rings=r)`` over fixed neighbour tables;
* device coordinates: shape, dtype, strides, device mismatch, never converted on the host (fake CUDA Array Interface objects).
"""

from __future__ import annotations

import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
from scipy.spatial import cKDTree
from sklearn.metrics.pairwise import cosine_similarity

from squidpy_b200.gr import _build as B


# ---- percentile ---------------------------------------------------------------------------------------------------------
def _percentile_two_stats(sorted_tail: np.ndarray, zeros: int, q: float) -> float:
    """``percentile_linear`` of graph_device.cu: m = zeros + len(sorted_tail) values, the zeros first."""
    m = zeros + sorted_tail.size
    get = lambda i: 0.0 if i < zeros else float(sorted_tail[i - zeros])  # noqa: E731
    vi = (m - 1) * (q / 100.0)
    prev = np.floor(vi)
    ip = int(prev)
    inx = ip + 1
    if vi >= m - 1:
        ip = inx = m - 1
        prev = -1.0
    gamma = vi - prev
    a, b = get(ip), get(inx)
    diff = b - a
    r = a + diff * gamma
    if gamma >= 0.5:
        r = b - diff * (1.0 - gamma)
    return r


def test_percentile_from_two_order_statistics_equals_numpy():
    rng = np.random.default_rng(0)
    qs = [0.0, 0.1, 1.0, 12.5, 33.3, 37.5, 49.999, 50.0, 50.001, 66.7, 90.0, 95.5, 99.0, 99.9, 100.0] + list(rng.random(40) * 100)
    for trial in range(40):
        m = int(rng.integers(1, 400))
        zeros = int(rng.integers(0, 50))
        d = np.round(rng.random(m) * 20.0, int(rng.integers(0, 4)))  # ties (and zeros) by rounding
        d[rng.random(m) < 0.1] = 0.0
        full = np.concatenate([np.zeros(zeros), d])
        rng.shuffle(full)
        for q in qs:
            got = _percentile_two_stats(np.sort(d), zeros, float(q))
            exp = np.percentile(full, q)
            assert got == exp, (trial, q, got, exp)


# ---- cosine -------------------------------------------------------------------------------------------------------------
def _cosine_restated(a: sp.csr_matrix) -> sp.csr_matrix:
    n = a.shape[0]
    x = a.data.astype(np.float32).copy()
    for r in range(n):
        s = 0.0
        for t in range(a.indptr[r], a.indptr[r + 1]):
            s += float(np.float32(x[t] * x[t]))
        if s == 0.0:
            continue
        s = np.sqrt(s)
        for t in range(a.indptr[r], a.indptr[r + 1]):
            x[t] = np.float32(np.float64(x[t]) / s)
    bt = sp.csr_matrix((x, a.indices, a.indptr), shape=a.shape).T.tocsr()
    bt.sort_indices()
    ptr, cols, vals = [0], [], []
    for r in range(n):
        # the products of the row in walk order, stably sorted by column, summed in order per column
        keys, prods = [], []
        for t in range(a.indptr[r], a.indptr[r + 1]):
            j, v = a.indices[t], x[t]
            for q in range(bt.indptr[j], bt.indptr[j + 1]):
                keys.append(bt.indices[q])
                prods.append(np.float32(v * bt.data[q]))
        order = np.argsort(np.asarray(keys, dtype=np.int64), kind="stable")
        q = 0
        while q < order.size:
            c, s = keys[order[q]], np.float32(0.0)
            while q < order.size and keys[order[q]] == c:
                s = np.float32(s + prods[order[q]])
                q += 1
            if s != 0:
                cols.append(c)
                vals.append(s)
        ptr.append(len(cols))
    return sp.csr_matrix((np.asarray(vals, np.float32), np.asarray(cols, np.int32), np.asarray(ptr, np.int32)), shape=a.shape)


def _knn_table(xy, k):
    d, i = cKDTree(xy).query(xy, k + 1)
    d, i = d[:, 1:], i[:, 1:].astype(np.int32)
    o = np.argsort(i, axis=1)
    return np.take_along_axis(d, o, 1), np.take_along_axis(i, o, 1)


@pytest.mark.parametrize("weights", ["unit", "random"])
def test_cosine_restatement_equals_sklearn(weights):
    rng = np.random.default_rng(1)
    xy = rng.random((300, 2)) * 100.0
    _, i = _knn_table(xy, 6)
    n = xy.shape[0]
    a = sp.csr_matrix((np.ones(i.size, np.float32), i.ravel(), np.arange(0, i.size + 1, 6, dtype=np.int32)), shape=(n, n))
    if weights == "random":
        a.data = rng.random(a.data.size).astype(np.float32)
    ref = cosine_similarity(a, dense_output=False).tocsr()
    ref.sort_indices()
    got = _cosine_restated(a)
    assert np.array_equal(ref.indptr, got.indptr) and np.array_equal(ref.indices, got.indices)
    assert ref.dtype == got.dtype and ref.data.tobytes() == got.data.tobytes()


def test_cosine_restatement_equals_host_builder_with_diagonal_and_percentile(monkeypatch):
    rng = np.random.default_rng(2)
    xy = rng.random((250, 2)) * 50.0
    d, i = _knn_table(xy, 5)
    monkeypatch.setattr(B, "knn_2d", lambda c, k, median=False, ctx=None: (d, i, np.median(d)) if median else (d, i))
    for kw in (dict(set_diag=True), dict(percentile=80.0), dict(set_diag=True, percentile=60.0)):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            host = B.KNNBuilder(5, transform="cosine", **kw).build(xy)[0].tocsr()
            plain = B.KNNBuilder(5, **kw).build(xy)[0].tocsr()
        host.sort_indices()
        plain.sort_indices()
        got = _cosine_restated(plain)
        assert np.array_equal(host.indptr, got.indptr) and np.array_equal(host.indices, got.indices)
        assert host.data.tobytes() == got.data.tobytes()


# ---- rings --------------------------------------------------------------------------------------------------------------
def _rings_restated(cut: sp.csr_matrix, n_rings: int) -> dict[tuple[int, int], int]:
    """graph_device.cu's level-by-level expansion: the level-d entries expand along the cut graph; a candidate already
    present keeps its level; the diagonal is dropped."""
    res = {(r, c): 1 for r in range(cut.shape[0]) for c in cut.indices[cut.indptr[r]:cut.indptr[r + 1]]}
    for level in range(1, n_rings):
        new = {}
        for (r, c), lv in res.items():
            if lv == level:
                for j in cut.indices[cut.indptr[c]:cut.indptr[c + 1]]:
                    if j != r and (r, j) not in res:
                        new[(r, int(j))] = level + 1
        if not new:
            break
        res.update(new)
    return res


@pytest.mark.parametrize("n_rings", [2, 3, 4])
@pytest.mark.parametrize("set_diag", [False, True])
def test_ring_levels_equal_grid_builder(monkeypatch, n_rings, set_diag):
    rng = np.random.default_rng(3)
    xy = rng.random((300, 2)) * 20.0
    d, i = _knn_table(xy, 6)
    monkeypatch.setattr(B, "knn_2d", lambda c, k, median=False, ctx=None: (d, i, np.median(d)) if median else (d, i))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        adj, dst = B.GridBuilder(6, n_rings=n_rings, set_diag=set_diag).build(xy)
        cut = B.GridBuilder(6).build(xy)[0].tocsr()
    cut.sort_indices()
    exp = _rings_restated(cut, n_rings)
    dst, adj = dst.tocsr(), adj.tocsr()
    rows = np.repeat(np.arange(dst.shape[0]), np.diff(dst.indptr))
    assert dict(zip(zip(rows.tolist(), dst.indices.tolist()), dst.data.tolist())) == {k: float(v) for k, v in exp.items()}
    assert dst.dtype == np.float32 and (adj.data == 1.0).all() and adj.dtype == np.float32
    assert adj.nnz == len(exp) + (adj.shape[0] if set_diag else 0)
    assert (adj.diagonal() == float(set_diag)).all()


# ---- device coordinate parsing ------------------------------------------------------------------------------------------
class FakeCoords:
    """A CUDA Array Interface exporter that is never converted on the host."""

    def __init__(self, shape, typestr="<f8", strides=None, ptr=0x7000_0000, stream=None):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3, "strides": strides, "stream": stream}

    def __array__(self, *a, **k):
        raise AssertionError("device coordinates were converted on the host")


def test_device_coordinates_are_parsed_not_converted():
    d = B._device_coords(FakeCoords((10, 2), strides=(48, 16), stream=5))
    assert d.shape == (10, 2) and d.strides == (6, 2) and d.dtype == np.float64 and d.stream == 5
    d = B._device_coords(FakeCoords((10, 2), typestr="<f4"))
    assert d.dtype == np.float32 and d.strides == (2, 1)
    assert B._device_coords(np.zeros((10, 2))) is None
    with pytest.raises(ValueError, match=r"shape `\(n, 2\)`"):
        B._device_coords(FakeCoords((10, 3)))
    with pytest.raises(ValueError, match=r"shape `\(n, 2\)`"):
        B._device_coords(FakeCoords((20,)))
    with pytest.raises(TypeError, match="float32 or float64"):
        B._device_coords(FakeCoords((10, 2), typestr="<i4"))
    with pytest.raises(ValueError, match="multiples of the item size"):
        B._device_coords(FakeCoords((10, 2), strides=(12, 4)))


def test_device_mismatch_raises_before_any_work(monkeypatch):
    monkeypatch.setattr(B, "pointer_device", lambda p: 0)
    monkeypatch.setattr(B, "load", lambda: (_ for _ in ()).throw(AssertionError("the library was called")))
    d = B._device_coords(FakeCoords((10, 2)))
    with pytest.raises(ValueError, match=r"`device=1` does not match the device of the spatial coordinates, cuda:0"):
        B.KNNBuilder(3).build_device(d, device=1)


def test_library_rows_follow_the_categories():
    from squidpy_b200 import AnnDataLite

    codes = np.array([2, 0, -1, 1, 0, 2, 2, 1])
    obs = pd.DataFrame({"lib": pd.Categorical.from_codes(codes, categories=["a", "b", "c"])}, index=[str(i) for i in range(8)])
    ptr, rows = B._library_rows(AnnDataLite(obs=obs, obsm={}, shape=(8, 0)), "lib")
    assert ptr.tolist() == [0, 2, 4, 7] and rows.dtype == np.int32
    assert [rows[ptr[b]:ptr[b + 1]].tolist() for b in range(3)] == [np.where(codes == b)[0].tolist() for b in range(3)]
