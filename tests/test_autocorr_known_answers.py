"""Moran's I / Geary's C pinned to the published definition (the reference's arithmetic lives in scanpy, which cannot be
imported here — SURVEY.md 8c): closed-form known answers, exact rational evaluation and a dense long-double third
formulation, applied to the CPU oracle (``-m "not gpu"``) and to the CUDA path through the C ABI (``-m gpu``)."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref
from tests import known_autocorr as ka

EXACT = dict(rtol=2e-14, atol=1e-15)  # float64 evaluation of a 5..36-node case against the correctly rounded value


def _random_asymmetric(seed=5, n=12):
    rng = np.random.default_rng(seed)
    m = (rng.random((n, n)) < 0.3) * rng.random((n, n))
    m[3, :] = 0.0  # a row without entries
    w = sp.csr_matrix(m.astype(np.float32))
    x = rng.normal(size=(4, n)).astype(np.float32)
    x[1, rng.random(n) < 0.6] = 0.0  # a sparse feature
    return w, x


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle restatement against sources it does not share code with
# ---------------------------------------------------------------------------------------------------------------------
def test_five_node_literals_are_exact():
    g, x = ka.five_node_asymmetric()
    assert ka.exact_autocorr(g, x) == (ka.FIVE_NODE_I, ka.FIVE_NODE_C)
    assert g.data[0] == np.float32(1.0) / np.float32(3.0) and abs(g.sum() - 4.0) < 1e-6  # rows 0,1,2,4 sum to 1; row 3 is empty


@pytest.mark.parametrize("case", ka.CASES, ids=[c[0] for c in ka.CASES])
def test_closed_forms_exact_and_oracle(case):
    _, w, x, exp_i, exp_c = case
    np.testing.assert_allclose(ka.exact_autocorr(w, x), (exp_i, exp_c), rtol=1e-15, atol=0)  # the derivation is right
    np.testing.assert_allclose(ka.dense_longdouble(w, x), (exp_i, exp_c), **EXACT)
    for vals in (x[None, :], sp.csr_matrix(x[None, :])):
        np.testing.assert_allclose(ref.morans_i(w, vals)[0], exp_i, **EXACT)
        np.testing.assert_allclose(ref.gearys_c(w, vals)[0], exp_c, **EXACT)


def test_oracle_vs_exact_on_random_asymmetric_graph():
    w, x = _random_asymmetric()
    exp = np.array([ka.exact_autocorr(w, row) for row in x])
    np.testing.assert_allclose(ref.morans_i(w, x), exp[:, 0], rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(ref.gearys_c(w, x), exp[:, 1], rtol=1e-13, atol=1e-15)


def test_oracle_vs_longdouble_on_dummy_adata(golden_dummy):
    """200 observations x 100 genes of the reference's ``dummy_adata`` recipe, raw and float32 row-normalised graph."""
    from sklearn.preprocessing import normalize

    g = sp.csr_matrix((golden_dummy["adj_data"], golden_dummy["adj_indices"], golden_dummy["adj_indptr"]), shape=(200, 200))
    gn = g.astype(np.float32).copy()
    normalize(gn, norm="l1", axis=1, copy=False)
    X = golden_dummy["X"]
    for w in (g, gn):
        exp = np.array([ka.dense_longdouble(w, X[:, k]) for k in range(X.shape[1])])
        np.testing.assert_allclose(ref.morans_i(w, X.T), exp[:, 0], rtol=1e-11, atol=1e-14)
        np.testing.assert_allclose(ref.gearys_c(w, X.T), exp[:, 1], rtol=1e-11, atol=1e-14)


def test_constant_feature_is_nan():
    w = ka.path_graph(10)
    assert np.isnan(ref.morans_i(w, np.full((1, 10), 2.5))).all() and np.isnan(ref.gearys_c(w, np.zeros((1, 10)))).all()


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the scalable long-double reference the GPU conditioning suite compares with
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("offset", [0.0, 1e2, 1e6, 1e12])
def test_sparse_longdouble_vs_exact(offset):
    """The closed-form cases, the asymmetric graphs (an empty row, an isolated source) and a feature far from 0 (the exact
    value of the definition does not care where the mean lies; a float64 evaluation does)."""
    cases = [(w, x) for _, w, x, _, _ in ka.CASES]
    w, x = _random_asymmetric()
    cases += [(w, row) for row in x] + [(w.astype(np.float64) * 0.7, x[2])]
    for w, x in cases:
        xo = np.asarray(x, dtype=np.float64) + offset
        exp = ka.exact_autocorr(w, xo)
        np.testing.assert_allclose(ka.sparse_longdouble(w, xo), exp, rtol=1e-15, atol=1e-16)
        si, sc = ka.autocorr_scale(w, xo)
        assert si >= abs(exp[0]) * (1 - 1e-12) and sc >= abs(exp[1]) * (1 - 1e-12)  # the scale bounds the value itself


def test_sparse_longdouble_vs_dense_on_dummy_adata(golden_dummy):
    from sklearn.preprocessing import normalize

    g = sp.csr_matrix((golden_dummy["adj_data"], golden_dummy["adj_indices"], golden_dummy["adj_indptr"]), shape=(200, 200))
    gn = g.astype(np.float32).copy()
    normalize(gn, norm="l1", axis=1, copy=False)
    X = golden_dummy["X"]
    for w in (g, gn):
        for k in range(X.shape[1]):
            np.testing.assert_allclose(ka.sparse_longdouble(w, X[:, k]), ka.dense_longdouble(w, X[:, k]), rtol=1e-15, atol=1e-17)


@pytest.mark.parametrize("value", [0.1, float(np.float32(0.1)), 1.0 / 3.0, -7.3, 0.0, 3.25])
def test_sparse_longdouble_constant_is_nan(value):
    w = ka.torus_grid(6)
    assert np.isnan(ka.sparse_longdouble(w, np.full(36, value))).all()
    x = np.full(36, value)
    x[7] = np.nextafter(value, np.inf)  # one ulp away: no longer constant, the definition is finite
    assert np.isfinite(ka.sparse_longdouble(w, x)).all()


def test_sparse_longdouble_million_observations_is_fast():
    import time

    from tools import synth

    g = synth.hex_graph(1000, 1000)
    x = 1e6 + np.random.default_rng(0).normal(size=g.shape[0])
    t = time.perf_counter()
    i, c = ka.sparse_longdouble(g, x)
    assert time.perf_counter() - t < 30.0
    assert abs(i) < 0.01 and abs(c - 1.0) < 0.01  # white noise: I ~ -1/(N-1), C ~ 1


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the CUDA kernels (dense tiles and the sparse per-feature kernel) against the same known answers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("case", ka.CASES, ids=[c[0] for c in ka.CASES])
def test_gpu_closed_forms(case, dtype):
    from squidpy_b200.gr import AutocorrPlan

    _, w, x, exp_i, exp_c = case
    plan = AutocorrPlan(w)
    xo = np.ascontiguousarray(x.astype(dtype)[:, None])  # observations x 1 feature
    for m in (xo, sp.csr_matrix(xo), sp.csr_matrix(xo.T)):
        plan.load(m, obs_major=(m.shape[0] == w.shape[0]))
        np.testing.assert_allclose(plan.score("moran")[0], exp_i, **EXACT)
        np.testing.assert_allclose(plan.score("geary")[0], exp_c, **EXACT)
    plan.close()


@pytest.mark.gpu
def test_gpu_vs_exact_on_random_asymmetric_graph():
    from squidpy_b200.gr import AutocorrPlan

    w, x = _random_asymmetric()
    exp = np.array([ka.exact_autocorr(w, row) for row in x])
    plan = AutocorrPlan(w)
    for m, om in ((x, False), (sp.csr_matrix(x), False), (sp.csr_matrix(x.T), True), (np.ascontiguousarray(x.T), True)):
        plan.load(m, obs_major=om)
        np.testing.assert_allclose(plan.score("moran"), exp[:, 0], rtol=1e-13, atol=1e-15)
        np.testing.assert_allclose(plan.score("geary"), exp[:, 1], rtol=1e-13, atol=1e-15)
    plan.close()


@pytest.mark.gpu
def test_gpu_vs_longdouble_on_dummy_adata(golden_dummy):
    from sklearn.preprocessing import normalize

    from squidpy_b200.gr import AutocorrPlan

    g = sp.csr_matrix((golden_dummy["adj_data"], golden_dummy["adj_indices"], golden_dummy["adj_indptr"]), shape=(200, 200))
    gn = g.astype(np.float32).copy()
    normalize(gn, norm="l1", axis=1, copy=False)
    X = golden_dummy["X"]
    for w in (g, gn):
        exp = np.array([ka.dense_longdouble(w, X[:, k]) for k in range(X.shape[1])])
        plan = AutocorrPlan(w)
        for m in (X, sp.csr_matrix(X)):
            plan.load(m, obs_major=True)
            np.testing.assert_allclose(plan.score("moran"), exp[:, 0], rtol=1e-11, atol=1e-14)
            np.testing.assert_allclose(plan.score("geary"), exp[:, 1], rtol=1e-11, atol=1e-14)
        plan.close()
