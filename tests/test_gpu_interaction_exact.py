"""interaction_matrix equals the reference bit for bit: every result, counts and weighted sums, host and device graphs, has the
oracle's dtype and bytes (the oracle is pinned to the reference in test_interaction_golden.py).  The oracle runs on the scipy
CSR of the graph as ``as_csr`` makes it, so a CSC graph is summed in the order of its ``tocsr()``: rows ascending, columns
ascending within a row, duplicates in storage order.  Each weighted float result is computed twice and must not change.

NaN is compared as NaN: which NaN bits an invalid operation produces differs between CPUs and GPUs and is no part of the
result (numpy does not define it either); every other value, -0.0 included, is compared by its bits."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from oracle import ref  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from tests.test_gpu_nhood_device_graph import CuSparse  # noqa: E402
from tests.test_interaction_golden import CASES, IDS  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu
FLAGS = [(False, False), (True, False), (False, True), (True, True)]  # (weights, normalized)
IDX = {"32": np.int32, "64": np.int64}
# host: scipy CSR / CSC; device: torch sparse_csr / sparse_csc (int64 indices) and cupy-style CSR / CSC with int32 or int64
# indptr and indices chosen independently
FORMS = ["host_csr", "host_csc", "torch_csr", "torch_csc"] + [f"cu_{f}_{p}_{i}" for f in ("csr", "csc") for p in IDX for i in IDX]
DEVICE_DTYPES = {np.dtype(t) for t in (np.float16, np.float32, np.float64, np.int32, np.int64, np.bool_)}


def _adata(g, codes, n_cats):
    cat = pd.Categorical.from_codes(np.asarray(codes), categories=[f"c{i}" for i in range(n_cats)])
    n = len(codes)
    return AnnDataLite(obs=pd.DataFrame({"cl": cat}, index=[str(i) for i in range(n)]), obsp={"spatial_connectivities": g}, shape=(n, 1))


def _call(g, codes, n_cats, weights, normalized):
    with np.errstate(divide="ignore", invalid="ignore"):
        return sq.gr.interaction_matrix(_adata(g, codes, n_cats), "cl", weights=weights, normalized=normalized, copy=True)


def _bits(a):
    a = np.array(a)
    if a.dtype.kind == "f":
        a[np.isnan(a)] = np.nan  # one NaN
    return a.tobytes()


def assert_exact(got, exp, what=""):
    assert got.dtype == exp.dtype, what
    assert got.shape == exp.shape, what
    if _bits(got) != _bits(exp):
        g, e = np.frombuffer(_bits(got), np.uint8).reshape(got.size, -1), np.frombuffer(_bits(exp), np.uint8).reshape(exp.size, -1)
        diff = np.flatnonzero((g != e).any(1))
        raise AssertionError(f"{what}: {diff.size} of {got.size} cells differ, first {diff[:4]}: got {got.ravel()[diff[:4]]!r}, "
                             f"expected {exp.ravel()[diff[:4]]!r}")


def make_form(g, form, data=None):
    """(graph in form ``form``, scipy CSR the oracle sums) of the CSR ``g``.  ``data``: float16 values in ``g``'s storage order
    for the device graph (scipy has no float16 matrices: the oracle sums their float64 twins)."""
    if data is not None:  # carried through the format change as positions
        g = sp.csr_matrix((np.arange(g.nnz, dtype=np.int64), g.indices, g.indptr), shape=g.shape)
    m = g.tocsc() if "csc" in form else g  # scipy keeps duplicates, in storage order
    vals = m.data if data is None else data[m.data]
    twin = m.copy()
    twin.data = vals.astype(np.float64) if data is not None else twin.data
    oracle = sp.csr_matrix(twin)
    if form.startswith("host"):
        assert data is None
        return m, oracle
    if form.startswith("torch"):
        ip, ix = (torch.from_numpy(a.astype(np.int64)) for a in (m.indptr, m.indices))
        make = torch.sparse_csr_tensor if m.format == "csr" else torch.sparse_csc_tensor
        return make(ip, ix, torch.from_numpy(np.ascontiguousarray(vals)), size=m.shape).cuda(), oracle
    _, _, p, i = form.split("_")
    return CuSparse(m.format, m.indptr.astype(IDX[p]), m.indices.astype(IDX[i]), vals, m.shape), oracle


def check_all(graph, oracle_csr, codes, n_cats, what="", flags=FLAGS):
    """Every (weights, normalized) of ``graph`` against the oracle on ``oracle_csr``; weighted float results twice."""
    for weights, normalized in flags:
        with np.errstate(divide="ignore", invalid="ignore"):
            exp = ref.interaction_matrix(oracle_csr, codes, n_cats, weights=weights, normalized=normalized)
        got = _call(graph, codes, n_cats, weights, normalized)
        assert_exact(got, exp, f"{what} weights={weights} normalized={normalized}")
        if weights and oracle_csr.dtype.kind == "f":
            again = _call(graph, codes, n_cats, weights, normalized)
            assert _bits(again) == _bits(got), f"{what}: a second run gave other bits"


# ---- the reference's fixtures ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_golden_cases(case, form):
    name, g, codes, n_cats, _, exp = case
    if not form.startswith("host") and g.dtype not in DEVICE_DTYPES:
        pytest.skip("int8 / int16 values are host-only")
    graph, csr = make_form(g, form)
    if "csc" not in form:
        for (w, nz), e in exp.items():  # the oracle is pinned to these: the same bytes
            assert_exact(_call(graph, codes, n_cats, w, nz), e, f"{name} {form} weights={w} normalized={nz}")
    check_all(graph, csr, codes, n_cats, f"{name} {form}")


def test_host_and_device_agree_on_every_weighted_case():
    """The host path and the device path give the same bytes for every weighted fixture (CSR and CSC)."""
    for name, g, codes, n_cats, _, _ in CASES:
        for fmt in ("csr", "csc"):
            host = _call(g if fmt == "csr" else g.tocsc(), codes, n_cats, True, False)
            if g.dtype in DEVICE_DTYPES:
                dev = _call(make_form(g, f"torch_{fmt}")[0], codes, n_cats, True, False)
                assert dev.dtype == host.dtype and _bits(dev) == _bits(host), (name, fmt)


# ---- value dtypes ---------------------------------------------------------------------------------------------------
def _values(dtype, size, rng):
    dtype = np.dtype(dtype)
    if dtype == np.float64:
        return rng.standard_normal(size) * 10.0 ** rng.integers(-12, 17, size)
    if dtype == np.float32:
        return (rng.standard_normal(size) * 10.0 ** rng.integers(-20, 20, size)).astype(np.float32)
    if dtype == np.float16:
        return (rng.standard_normal(size) * 2.0 ** rng.integers(-24, 12, size)).astype(np.float16)
    if dtype == np.int64:
        return ((rng.integers(0, 2, size) * 2 - 1) * (2**62 - rng.integers(0, 99, size))).astype(np.int64)
    if dtype == np.int32:
        return rng.integers(-(2**31), 2**31, size).astype(np.int32)
    return rng.random(size) < 0.6


@pytest.mark.parametrize("form", ["host_csr", "host_csc", "torch_csr", "torch_csc", "cu_csr_64_32", "cu_csc_32_64"])
@pytest.mark.parametrize("dtype", ["float32", "float64", "float16", "int32", "int64", "bool"])
def test_value_dtypes(dtype, form):
    rng = np.random.default_rng(7)
    g = synth.knn_graph(rng.random((3000, 2)) * 100, k=9)
    g = sp.csr_matrix((_values(dtype, g.nnz, rng), g.indices, g.indptr), shape=g.shape) if dtype != "float16" else g
    codes = rng.integers(-1, 7, g.shape[0])
    if dtype == "float16" and form.startswith("host"):
        pytest.skip("float16 graphs are device-only")
    graph, csr = make_form(g, form, _values(np.float16, g.nnz, rng) if dtype == "float16" else None)
    check_all(graph, csr, codes, 7, f"{dtype} {form}")


# ---- kernel edges ---------------------------------------------------------------------------------------------------
def _edge_graph(kind, rng):
    if kind == "many_rows":  # more rows than warps in the grid (8 blocks of 8 warps per SM): the row loop wraps
        g = synth.knn_graph(rng.random((20000, 2)) * 400, k=5)
    elif kind == "long_rows":  # rows of up to 150 entries: one row spans several strides of the 32 lanes
        n = 2500
        lens = rng.integers(0, 150, n)
        ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        g = sp.csr_matrix((np.ones(ptr[-1]), rng.integers(0, n, ptr[-1]), ptr), shape=(n, n))
    else:
        assert kind == "nnz0"
        return sp.csr_matrix((500, 500), dtype=np.float64)
    return sp.csr_matrix((_values(np.float64, g.nnz, rng), g.indices, g.indptr), shape=g.shape)


@pytest.mark.parametrize("n_cats", [1, 2, 78, 79, 4096])  # 78 / 79: either side of C*C*8 <= 48 KiB (shared-memory bins)
@pytest.mark.parametrize("kind", ["many_rows", "long_rows", "nnz0"])
def test_kernel_edges(kind, n_cats):
    rng = np.random.default_rng(n_cats)
    g = _edge_graph(kind, rng)
    n = g.shape[0]
    codes = rng.integers(0, n_cats, n)
    if n_cats > 2:
        codes[codes == n_cats // 2] = n_cats - 1  # a category with no members
    codes[rng.random(n) < 0.05] = -1
    if not (codes >= 0).any():
        codes[0] = 0
    for form in ("host_csr", "torch_csr", "cu_csc_64_32"):
        for dtype in (np.float64, np.float32, np.int64):
            gd = sp.csr_matrix((_values(dtype, g.nnz, rng) if g.nnz else g.data.astype(dtype), g.indices, g.indptr), shape=g.shape)
            graph, csr = make_form(gd, form)
            check_all(graph, csr, codes, n_cats, f"{kind} C={n_cats} {form} {np.dtype(dtype).name}")
    for form in ("host_csr", "torch_csc"):  # binary weights (weights=True on a connectivity graph)
        graph, csr = make_form(sp.csr_matrix((np.ones(g.nnz, np.float32), g.indices, g.indptr), shape=g.shape), form)
        check_all(graph, csr, codes, n_cats, f"{kind} C={n_cats} {form} binary", flags=[(True, False), (True, True)])


def test_rows_summing_to_zero_normalize_to_nan():
    """normalized=True divides every row by its sum; a row summing to exactly 0 gives NaN (0 / 0) or ±inf, as numpy does."""
    g = sp.csr_matrix((np.array([1e16, -1e16, 1.0, -1.0, 2.0, 0.5]), np.array([1, 2, 0, 3, 2, 0]), np.array([0, 2, 4, 5, 6, 6])),
                      shape=(5, 5))
    codes = np.array([0, 1, 1, 2, 2])
    for form in ("host_csr", "torch_csr", "cu_csc_32_32"):
        graph, csr = make_form(g, form)
        got = _call(graph, codes, 4, True, True)
        assert np.isnan(got[0]).all() and np.isnan(got[3]).all()  # row 0: 1e16 - 1e16; row 3: no entries
        check_all(graph, csr, codes, 4, form)


# ---- scale ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", ["host_csr", "torch_csr", "cu_csc_32_32"])
def test_million_cells_two_categories(form):
    """1000 x 1000 hex graph (6 M entries), random float32 weights, C = 2: every cell is a chain of ~1.5 M additions."""
    g = synth.hex_graph(1000, 1000)
    rng = np.random.default_rng(11)
    g = sp.csr_matrix((rng.random(g.nnz).astype(np.float32), g.indices, g.indptr), shape=g.shape)  # not on a 2^-24 grid
    codes = rng.integers(0, 2, g.shape[0])
    codes[rng.random(g.shape[0]) < 0.01] = -1
    graph, csr = make_form(g, form)
    check_all(graph, csr, codes, 2, form, flags=[(True, False), (True, True)])
