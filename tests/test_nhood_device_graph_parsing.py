"""Host logic of device-resident neighbour graphs (no GPU, no library call): graph-format detection, the index-width codes
and sizes handed to the C ABI, the transposition that turns the results of a CSC graph back into the graph's, and the
guarantee that a device graph never goes through scipy (``as_csr``) on its way to nhood_enrichment / interaction_matrix."""

from __future__ import annotations

import threading

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

from squidpy_b200 import AnnDataLite
from squidpy_b200._device import GRAPH_VALUE_CODES, DevGraph, device_graph, graph_args, graph_value_code, parse_cai
from squidpy_b200.gr import _nhood

KEY = "spatial_connectivities"


class FakeDev:
    """An object exposing a hand-written __cuda_array_interface__; reading it on the host fails."""

    def __init__(self, shape, typestr, ptr, stream=None, strides=None):
        self.shape = tuple(shape)
        self.__cuda_array_interface__ = dict(shape=self.shape, typestr=typestr, data=(ptr, False), strides=strides, version=3, stream=stream)

    def __array__(self, *a, **k):
        raise AssertionError("__array__ called on a device array")


class FakeGraph:
    """cupyx-style device CSR / CSC graph of n x n with nnz stored entries."""

    def __init__(self, fmt, n=6, nnz=9, ip="<i4", ix="<i4", val="<f4", stream=None, shape=None, n_ptr=None):
        self.format, self.shape = fmt, shape or (n, n)
        self.indptr = FakeDev(((n + 1) if n_ptr is None else n_ptr,), ip, 0x1000, stream)
        self.indices = FakeDev((nnz,), ix, 0x2000 if nnz else 0, stream)
        self.data = FakeDev((nnz,), val, 0x3000 if nnz else 0, stream)

    def __array__(self, *a, **k):
        raise AssertionError("__array__ called on a device graph")


def test_graph_format_detection():
    assert device_graph(sp.random(5, 5, density=0.3, format="csr")) is None
    assert device_graph(np.eye(4)) is None
    for fmt in ("csr", "csc"):
        d = device_graph(FakeGraph(fmt))
        assert d.format == fmt and d.shape == (6, 6)
    with pytest.raises(NotImplementedError, match="Dense device graphs.*csr, csc"):
        device_graph(FakeDev((6, 6), "<f4", 0x1000))
    g = FakeGraph("coo")
    with pytest.raises(NotImplementedError, match="csr, csc"):
        device_graph(g)


@pytest.mark.parametrize("ip, ix, bits", [("<i4", "<i4", (32, 32)), ("<i8", "<i8", (64, 64)), ("<i8", "<i4", (64, 32)), ("<i4", "<i8", (32, 64))])
@pytest.mark.parametrize("fmt", ["csr", "csc"])
def test_abi_arguments(ip, ix, bits, fmt):
    a = graph_args(device_graph(FakeGraph(fmt, n=6, nnz=9, ip=ip, ix=ix, stream=77)), 6)
    assert isinstance(a, DevGraph)
    assert (a.indptr_bits, a.index_bits) == bits
    assert (a.n, a.nnz, a.indptr, a.indices, a.stream) == (6, 9, 0x1000, 0x2000, 77)
    assert a.transposed == (fmt == "csc")  # a CSC graph is handed over as the CSR of its transpose


def test_abi_argument_errors():
    with pytest.raises(ValueError, match="shape"):
        graph_args(device_graph(FakeGraph("csr", n=6, shape=(6, 7))), 6)
    with pytest.raises(ValueError, match="shape"):
        graph_args(device_graph(FakeGraph("csr", n=6)), 7)  # the graph of another AnnData
    with pytest.raises(ValueError, match="indptr"):
        graph_args(device_graph(FakeGraph("csr", n=6, n_ptr=6)), 6)
    with pytest.raises(TypeError, match="int32 or int64"):
        graph_args(device_graph(FakeGraph("csr", ix="<u4")), 6)
    with pytest.raises(TypeError, match="int32 or int64"):
        graph_args(device_graph(FakeGraph("csr", ip="<f8")), 6)
    g = FakeGraph("csr")
    g.indices = FakeDev((9,), "<i4", 0x2000, strides=(8,))
    with pytest.raises(ValueError, match="contiguous"):
        graph_args(device_graph(g), 6)
    g = FakeGraph("csr", stream=5)
    g.data = FakeDev((9,), "<f4", 0x3000, stream=6)
    with pytest.raises(ValueError, match="different producer streams"):
        graph_args(device_graph(g), 6)
    e = graph_args(device_graph(FakeGraph("csr", nnz=0)), 6)  # an empty graph has no index allocation
    assert e.nnz == 0 and e.indices == 0


def test_value_codes():
    codes = {t: graph_value_code(parse_cai(FakeDev((4,), t, 0x10)), 4) for t in ("<f4", "<f8", "<f2", "<i4", "<i8", "|b1")}
    assert codes == {"<f4": 0, "<f8": 1, "<f2": 2, "<i4": 3, "<i8": 4, "|b1": 5}
    assert len(GRAPH_VALUE_CODES) == 6
    for t in ("<u1", "<i2", "<c8"):
        with pytest.raises(TypeError, match="not supported"):
            graph_value_code(parse_cai(FakeDev((4,), t, 0x10)), 4)
    with pytest.raises(ValueError, match="4"):
        graph_value_code(parse_cai(FakeDev((3,), "<f4", 0x10)), 4)


def _adata(graph, n=6, n_cls=3):
    labels = np.arange(n) % n_cls
    obs = pd.DataFrame({"cl": pd.Categorical.from_codes(labels, categories=[f"c{i}" for i in range(n_cls)])}, index=[str(i) for i in range(n)])
    return AnnDataLite(obs=obs, obsp={KEY: graph}, shape=(n, 1))


class _Ctx:
    device = 0
    handle = None
    lock = threading.RLock()


class _FakePlan:
    """Stands in for the device plan of a CSC graph: it holds the transpose, so its results are transposes too."""

    count_t = np.array([[5, 1, 0], [7, 2, 3], [0, 9, 4]], dtype=np.uint32)
    mean_t = np.array([[2.0, 0.5, 0.25], [3.0, 1.0, 2.0], [0.5, 4.0, 1.5]])
    std_t = np.array([[1.0, 0.5, 0.5], [2.0, 1.0, 1.0], [0.25, 2.0, 0.5]])

    def count(self, labels):
        return self.count_t.copy()

    def set_base(self, *a):
        pass

    def upload_philox(self, *a):
        pass

    def run_async(self):
        pass

    def stats(self):
        return self.mean_t.copy(), self.std_t.copy()

    def close(self):
        pass


@pytest.fixture()
def no_scipy_graph(monkeypatch):
    """Device graphs must reach the library without as_csr; the context is a stand-in and the device lookup is skipped."""

    def fail(*a, **k):
        raise AssertionError("a device graph was converted by as_csr")

    monkeypatch.setattr(_nhood, "as_csr", fail)
    monkeypatch.setattr(_nhood, "_graph_device", lambda d, device: 0)
    monkeypatch.setattr(_nhood, "default_context", lambda device=None: _Ctx())


@pytest.mark.parametrize("fmt", ["csr", "csc"])
def test_nhood_csc_transposes_count_mean_and_std(no_scipy_graph, monkeypatch, fmt):
    seen = {}

    def from_device(graph, n_cls, ctx):
        seen["graph"] = graph
        return _FakePlan()

    monkeypatch.setattr(_nhood.NhoodPlan, "from_device", staticmethod(from_device))
    res = _nhood.nhood_enrichment(_adata(FakeGraph(fmt)), "cl", n_perms=4, seed=0, copy=True, rng="philox")
    assert seen["graph"].transposed == (fmt == "csc")
    P = _FakePlan
    t = (lambda a: a.T) if fmt == "csc" else (lambda a: a)
    assert np.array_equal(res.counts, t(P.count_t)) and res.counts.flags.c_contiguous
    with np.errstate(divide="ignore", invalid="ignore"):
        assert np.array_equal(res.zscore, (t(P.count_t) - t(P.mean_t)) / t(P.std_t))


@pytest.mark.parametrize("weights", [False, True])
@pytest.mark.parametrize("fmt", ["csr", "csc"])
def test_interaction_passes_the_csc_flag_and_transposes_the_result(no_scipy_graph, monkeypatch, fmt, weights):
    block = np.array([[1, 2, 3], [4, 5, 6], [7, 8, 10]])
    calls = []

    class Lib:
        def sqb_interaction_matrix_device(self, ctx, n, nnz, ip, ip_bits, ix, ix_bits, csc, data, code, codes, n_cats, out_w, out_c, stream):
            calls.append((n, nnz, ip_bits, ix_bits, csc, data, code))
            import ctypes

            dst = out_w if weights else out_c
            arr = np.ctypeslib.as_array(ctypes.cast(dst, ctypes.POINTER(ctypes.c_double if weights else ctypes.c_int64)), shape=(n_cats, n_cats))
            arr[...] = block
            return 0

    monkeypatch.setattr(_nhood, "load", lambda: Lib())
    out = _nhood.interaction_matrix(_adata(FakeGraph(fmt, ip="<i8")), "cl", weights=weights, copy=True)
    assert calls == [(6, 9, 64, 32, int(fmt == "csc"), 0x3000 if weights else None, 0 if weights else -1)]
    assert out.dtype == np.float64  # float32 graph values: float64 as on the host
    assert np.array_equal(out, block.T if fmt == "csc" else block)


def test_interaction_output_dtype_follows_the_value_dtype(no_scipy_graph, monkeypatch):
    class Lib:
        def sqb_interaction_matrix_device(self, *a):
            return 0

    monkeypatch.setattr(_nhood, "load", lambda: Lib())
    for val, weights, dtype in (("|b1", False, np.int64), ("<i4", True, np.int64), ("<i8", False, np.int64), ("<f2", True, np.float64),
                                ("<f8", False, np.float64)):
        out = _nhood.interaction_matrix(_adata(FakeGraph("csr", val=val)), "cl", weights=weights, copy=True)
        assert out.dtype == dtype, (val, weights)
    with pytest.raises(TypeError, match="not supported"):
        _nhood.interaction_matrix(_adata(FakeGraph("csr", val="<u2")), "cl", weights=True, copy=True)


def test_dense_device_graph_is_refused():
    dense = FakeDev((6, 6), "<f4", 0x1000)
    with pytest.raises(NotImplementedError, match="csr, csc"):
        _nhood.nhood_enrichment(_adata(dense), "cl", n_perms=4, copy=True)
    with pytest.raises(NotImplementedError, match="csr, csc"):
        _nhood.interaction_matrix(_adata(dense), "cl", copy=True)
