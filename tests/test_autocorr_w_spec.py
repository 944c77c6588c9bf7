"""The specification of spatial_autocorr's device build of W (``tests/autocorr_w_ref.py``) against the libraries it restates:
sklearn's l1 ``normalize``, ``np.sum``, and ``_g_moments`` on scipy, bit for bit and with the same scalar types; and the
predicate that lets S0 be summed exactly in parallel.  CPU only."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

from squidpy_b200.gr._ppatterns import _g_moments
from tests import autocorr_w_ref as ref
from tools import synth

DTYPES = [np.float32, np.float64]


def _random_graph(n, max_deg, dtype, seed, *, signs=True, zeros=True, loops=True):
    """Canonical CSR with rows of 0..max_deg entries, mixed magnitudes and signs, explicit zeros and self-loops."""
    rng = np.random.default_rng(seed)
    ptr, idx, val = [0], [], []
    for r in range(n):
        d = int(rng.integers(0, max_deg + 1)) if r % 11 else 0
        cols = np.sort(rng.choice(n, size=min(d, n), replace=False))
        if loops and r % 5 == 0 and r not in cols:
            cols = np.sort(np.append(cols, r))
        v = rng.random(cols.size) * 10.0 ** rng.integers(-4, 4, cols.size)
        if signs:
            v *= rng.choice([-1.0, 1.0], cols.size)
        if zeros and cols.size:
            v[rng.random(cols.size) < 0.1] = 0.0
        idx += list(cols)
        val += list(v)
        ptr.append(len(idx))
    return sp.csr_matrix((np.asarray(val, dtype), np.asarray(idx, np.int32), np.asarray(ptr, np.int32)), shape=(n, n))


def _same(a, b):
    return type(a) is type(b) and np.asarray(a).tobytes() == np.asarray(b).tobytes()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("max_deg", [6, 40])
def test_l1_normalisation_equals_sklearn(dtype, max_deg):
    from sklearn.preprocessing import normalize

    g = _random_graph(600, max_deg, dtype, seed=max_deg)
    assert np.any(np.diff(g.indptr) == 0) and (max_deg < 16 or np.any(np.diff(g.indptr) > 16))
    assert np.any(g.data == 0) and np.any(g.data < 0) and np.any(g.diagonal() != 0)
    h = g.copy()
    normalize(h, norm="l1", axis=1, copy=False)
    got = ref.l1_normalize(g.indptr, g.data)
    assert got.dtype == h.data.dtype
    assert got.tobytes() == h.data.tobytes()


@pytest.mark.parametrize("dtype", DTYPES)
def test_pairwise_sum_equals_np_sum_every_length(dtype):
    rng = np.random.default_rng(1)
    for n in range(0, 1101):
        a = (rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)).astype(dtype)
        assert ref.np_sum(a).tobytes() == np.sum(a).tobytes(), n


@pytest.mark.parametrize("dtype", DTYPES)
def test_pairwise_sum_equals_np_sum_long(dtype):
    rng = np.random.default_rng(2)
    for n in [int(x) for x in rng.integers(1101, 10**7, 3)] + [10**7]:
        a = (rng.standard_normal(n) * 10.0 ** rng.integers(-6, 6, n)).astype(dtype)
        assert ref.np_sum(a).tobytes() == np.sum(a).tobytes(), n


def _graphs():
    hexg = synth.hex_graph(30, 40)
    knn = synth.knn_graph(synth.hex_coords(30, 40) + np.random.default_rng(0).normal(0, 7, (1200, 2)), k=6)
    yield "hex", hexg
    yield "knn", knn
    yield "knn_weighted", sp.csr_matrix((np.random.default_rng(3).random(knn.nnz).astype(np.float32), knn.indices, knn.indptr), shape=knn.shape)
    for dt in DTYPES:
        yield f"random_{np.dtype(dt).name}", _random_graph(700, 30, dt, seed=4)
        yield f"random_long_{np.dtype(dt).name}", _random_graph(300, 290, dt, seed=5)
        yield f"empty_{np.dtype(dt).name}", sp.csr_matrix((50, 50), dtype=dt)


@pytest.mark.parametrize("normalise", [False, True])
@pytest.mark.parametrize("name,g", list(_graphs()), ids=[n for n, _ in _graphs()])
def test_moments_equal_g_moments(name, g, normalise):
    from sklearn.preprocessing import normalize

    g = g.copy()
    g.sort_indices()
    if normalise:
        normalize(g, norm="l1", axis=1, copy=False)
    exp = _g_moments(g)
    got = ref.g_moments(g.shape[0], g.indptr, g.indices, g.data)
    for a, b in zip(got, exp):
        assert _same(a, b), (name, a, b, type(a), type(b))


def test_moments_with_cancelling_and_underflowing_entries():
    # w_ij + w_ji == 0 and squares below float32's range drop out of W + W^T and of its square: the sums' trees change
    n = 40
    rows, cols, vals = [], [], []
    for i in range(n - 1):
        rows += [i, i + 1]
        cols += [i + 1, i]
        v = np.float32(1e-24) if i % 4 == 0 else np.float32(i + 1)
        vals += [v, -v if i % 3 == 0 else v]
    g = sp.csr_matrix((np.asarray(vals, np.float32), (rows, cols)), shape=(n, n))
    g.sort_indices()
    exp = _g_moments(g)
    got = ref.g_moments(n, g.indptr, g.indices, g.data)
    for a, b in zip(got, exp):
        assert _same(a, b), (a, b)


@pytest.mark.parametrize("name,g", [(n, g) for n, g in _graphs() if n in ("hex", "knn", "knn_weighted")], ids=lambda x: x if isinstance(x, str) else "")
def test_s0_predicate_holds_on_row_normalised_graphs(name, g):
    from sklearn.preprocessing import normalize

    g = g.copy()
    normalize(g, norm="l1", axis=1, copy=False)
    wd = g.data.astype(np.float64)
    assert ref.s0_exact_predicate(wd)
    assert ref.s0_exact(wd) == ref.s0_sequential(wd)


def test_s0_predicate_fails_where_partial_sums_round():
    # 1 + 2^-53 rounds back to 1 twice, while the exact sum 1 + 2^-52 is representable: the integer sum would differ
    wd = np.array([1.0, 2.0**-53, 2.0**-53])
    assert not ref.s0_exact_predicate(wd)
    assert ref.s0_exact(wd) != ref.s0_sequential(wd)
    assert not ref.s0_exact_predicate(np.array([1.0, np.inf]))
    assert not ref.s0_exact_predicate(np.array([1.0, np.nan]))
    assert ref.s0_exact_predicate(np.zeros(3))
