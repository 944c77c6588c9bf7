"""sepal's saturation tables without a GPU: which inputs ``sepal_idxs`` hands to ``sqb_sepal_idxs`` and which take
``_compute_idxs`` on host copies, how the arguments are marshalled (the ABI replaced by a restatement that reads them back), and
the orphan rules of the host restatement and of the device reduction, pinned against scikit-learn and numpy."""

from __future__ import annotations

import ctypes as C
import threading

import numpy as np
import pytest
import scipy.sparse as sp
from scipy.spatial.distance import cdist
from sklearn.metrics import pairwise_distances

import squidpy_b200.gr._sepal as S
import squidpy_b200.gr._utils as U
from tools.sepal_idx_time import lattice

VALUE_DTYPES = {0: np.float32, 1: np.float64, 3: np.int32, 4: np.int64, 5: np.bool_}


def _expected(g, co, k):
    h = g.copy() if (sp.issparse(g) and g.format == "csr") else sp.csr_matrix(g)
    h.eliminate_zeros()
    return S._compute_idxs(h, np.asarray(co, dtype=np.float64), k)


def _read(ptr, dtype, count):
    dtype = np.dtype(dtype)
    if count == 0:
        return np.empty(0, dtype)
    return np.frombuffer((C.c_char * (count * dtype.itemsize)).from_address(ptr), dtype=dtype).copy()


def _write(ptr, arr):
    arr = np.ascontiguousarray(arr, dtype=np.int32)
    if arr.size:
        C.memmove(ptr, arr.ctypes.data, arr.nbytes)


class FakeLib:
    """``sqb_sepal_idxs`` restated on the host: host arrays are read back through their pointers, a device graph or coordinates
    are taken from ``twins`` (pointer -> host array).  Every call's arguments are recorded."""

    def __init__(self, twins=None, max_degree=None, nonfinite=None):
        self.calls, self.twins, self.max_degree, self.nonfinite = [], twins or {}, max_degree, nonfinite

    def sqb_sepal_idxs(self, handle, *a):
        (n, nnz, ip, ip_bits, ix, ix_bits, data, code, csc, dev_in, _, xy, xy_dtype, sr, sc, xy_dev, _, k, max_deg, sat, sat_idx, unsat, unsat_idx,
         n_sat, n_unsat, bad) = a
        self.calls.append(dict(zip(("n", "nnz", "indptr", "indptr_bits", "indices", "index_bits", "data", "data_dtype", "csc", "device_input",
                                    "producer_stream", "xy", "xy_dtype", "stride_row", "stride_col", "xy_device", "xy_stream", "max_neighs"), a[:18])))
        if dev_in:
            indptr, indices, values = self.twins[ip], self.twins[ix], self.twins[data]
        else:
            indptr, indices = _read(ip, f"int{ip_bits}", n + 1), _read(ix, f"int{ix_bits}", nnz)
            values = _read(data, VALUE_DTYPES[code], nnz)
        m = sp.csr_matrix((sp.csc_matrix if csc else sp.csr_matrix)((values, indices, indptr), shape=(n, n)))
        m.eliminate_zeros()
        most = int(np.diff(m.indptr).max()) if self.max_degree is None else self.max_degree
        max_deg._obj.value = most
        if most != k:
            return 0
        xy_host = self.twins[xy] if xy_dev else _read(xy, np.float64, 2 * n).reshape(n, 2)
        tables = S._compute_idxs(m, np.nan_to_num(np.asarray(xy_host, dtype=np.float64)), k)
        for ptr, arr in zip((sat, sat_idx, unsat, unsat_idx), tables):
            _write(ptr, arr.ravel())
        n_sat._obj.value, n_unsat._obj.value = tables[0].size, tables[2].size
        bad._obj.value = int(bool(self.nonfinite))
        return 0

    def sqb_last_error(self):
        return b"fake"


class FakeCtx:
    def __init__(self, device):
        self.device, self.handle, self.lock = device, None, threading.RLock()


class Dev:
    """A device array as the CUDA Array Interface describes it (the pointer is only a key of FakeLib.twins)."""

    _next = 0x10000

    def __init__(self, host, stream=None, strides=None, ptr=None):
        Dev._next += 0x10000
        self.host = np.asarray(host)
        self.ptr = Dev._next if ptr is None else ptr
        self.__cuda_array_interface__ = {"shape": self.host.shape, "typestr": self.host.dtype.str, "data": (self.ptr, False), "version": 3,
                                         "strides": strides, "stream": stream}
        self.shape = self.host.shape


class DevCsr:
    def __init__(self, m, ip=np.int32, ix=np.int32, stream=None):
        self.format, self.shape, self.host = m.format, m.shape, m
        self.indptr, self.indices, self.data = Dev(m.indptr.astype(ip), stream), Dev(m.indices.astype(ix), stream), Dev(m.data, stream)


@pytest.fixture
def fake(monkeypatch):
    """Installs a FakeLib; device pointers live on device 1 unless listed in ``where``; ``ctx`` records the devices asked for."""
    state = {"lib": FakeLib(), "ctx": [], "where": {}}

    def pointer_device(ptr):
        return state["where"].get(ptr, 1 if ptr >= 0x20000 else -1)

    def on_host(m):
        if isinstance(m, DevCsr):
            return m.host
        return m.host if isinstance(m, Dev) else m

    monkeypatch.setattr(S, "load", lambda: state["lib"])
    monkeypatch.setattr(S, "check", lambda rc: None)
    monkeypatch.setattr(S, "default_context", lambda device=None: state["ctx"].append(device) or FakeCtx(0 if device is None else device))
    monkeypatch.setattr(S, "pointer_device", pointer_device)
    monkeypatch.setattr(U, "pointer_device", pointer_device)
    monkeypatch.setattr(S, "on_host", on_host)
    return state


def _twins(state, *objs):
    for o in objs:
        for d in (o.indptr, o.indices, o.data) if isinstance(o, DevCsr) else (o,):
            state["lib"].twins[d.ptr] = d.host


@pytest.fixture(scope="module")
def case():
    g, co, k = lattice("square", 30, 0.15, seed=2)
    return g, co, k


@pytest.mark.parametrize("form", ["csr", "csr64", "csc", "dense", "coo", "int8", "bool", "float32_zeros"])
def test_host_graphs_take_the_device_path(fake, case, form):
    g, co, k = case
    m = {"csr": g, "csr64": g.astype(np.float64),
         "csc": sp.csc_matrix(g), "dense": g.toarray(), "coo": g.tocoo(), "int8": g.astype(np.int8), "bool": g.astype(bool)}.get(form)
    if form == "csr64":
        m.indices, m.indptr = m.indices.astype(np.int64), m.indptr.astype(np.int64)
    if form == "float32_zeros":
        m = g.copy()
        m.data[::7] = 0.0
        m.data[3::11] = -0.0
    got = S.sepal_idxs(m, co, k, device=0)
    for a, b in zip(got, _expected(m, co, k), strict=True):
        assert np.array_equal(a, b) and a.dtype == np.int32
    (call,) = fake["lib"].calls
    assert call["device_input"] == 0 and call["xy_device"] == 0 and (call["xy_dtype"], call["stride_row"], call["stride_col"]) == (1, 2, 1)
    assert call["csc"] == (form == "csc") and call["max_neighs"] == k and call["n"] == g.shape[0]
    assert call["data_dtype"] == {"csr64": 1, "int8": 5, "bool": 5}.get(form, 0)
    assert (call["indptr_bits"], call["index_bits"]) == ((64, 64) if form == "csr64" else (32, 32))
    assert fake["ctx"] == [0]


def test_other_host_value_dtypes_pass_their_non_zero_mask(fake, case):
    g, co, k = case
    m = g.astype(np.int8)
    m.data[::5] = 0
    m.data[1::5] = -3
    S.sepal_idxs(m, co, k)
    (call,) = fake["lib"].calls
    assert call["data_dtype"] == 5  # bool: what eliminate_zeros keeps


def test_copy_path_inputs(fake, case):
    g, co, k = case
    want = _expected(g, co, k)
    f16 = DevCsr(g)
    f16.data = Dev(g.data.astype(np.float16))  # scipy has no float16 matrices
    strided = DevCsr(g)
    strided.data.__cuda_array_interface__["strides"] = (2 * g.data.itemsize,)
    two_devices = DevCsr(g)
    fake["where"][two_devices.indices.ptr] = 2
    for conn, xy in ((g, np.c_[co, co[:, :1]]),  # coordinates that are not n x 2
                     (Dev(g.toarray()), co),  # a dense device graph
                     (f16, co), (strided, co), (two_devices, co)):  # float16 values, strided values, arrays on two devices
        got = S.sepal_idxs(conn, xy, k)
        ref = _expected(g, np.asarray(xy, dtype=np.float64), k)
        for a, b in zip(got, ref, strict=True):
            assert np.array_equal(a, b)
    assert not fake["lib"].calls
    assert all(np.array_equal(a, b) for a, b in zip(S.sepal_idxs(g, co, k), want))


def test_device_graph_arguments(fake, case):
    g, co, k = case
    conn = DevCsr(sp.csr_matrix(g), np.int64, np.int64, stream=7)
    xy = Dev(co.astype(np.float32), stream=9)
    _twins(fake, conn, xy)
    got = S.sepal_idxs(conn, xy, k, device=0)  # `device` names another GPU than the graph's: the graph's own is used
    for a, b in zip(got, _expected(g, co.astype(np.float32), k), strict=True):
        assert np.array_equal(a, b)
    (call,) = fake["lib"].calls
    assert fake["ctx"] == [1]
    assert (call["device_input"], call["indptr"], call["indices"], call["data"]) == (1, conn.indptr.ptr, conn.indices.ptr, conn.data.ptr)
    assert (call["indptr_bits"], call["index_bits"], call["data_dtype"], call["csc"], call["producer_stream"]) == (64, 64, 0, 0, 7)
    assert (call["xy"], call["xy_device"], call["xy_dtype"], call["stride_row"], call["stride_col"], call["xy_stream"]) == (xy.ptr, 1, 0, 2, 1, 9)


def test_device_csc_and_coordinates_elsewhere(fake, case):
    g, co, k = case
    conn = DevCsr(sp.csc_matrix(g), stream=None)
    conn.data = Dev(conn.host.data.astype(np.int64))
    f_order = Dev(co, strides=(8, 8 * co.shape[0]))  # read in place with element strides (1, n)
    other = Dev(co)
    fake["where"][other.ptr] = 3  # on another device: copied to the host
    half = Dev(co.astype(np.float16))
    _twins(fake, conn, f_order)
    for xy, dev, strides in ((f_order, 1, (1, co.shape[0])), (other, 0, (2, 1)), (half, 0, (2, 1))):
        fake["lib"].calls.clear()
        S.sepal_idxs(conn, xy, k)
        (call,) = fake["lib"].calls
        assert (call["csc"], call["data_dtype"], call["device_input"]) == (1, 4, 1)
        assert (call["xy_device"], (call["stride_row"], call["stride_col"])) == (dev, strides)


def test_max_neighs_error_and_nonfinite_fallback(fake, case):
    g, co, k = case
    fake["lib"].max_degree = 5
    with pytest.raises(ValueError, match=r"^Expected `max_neighs=4`, found node with `5` neighbors\.$"):
        S.sepal_idxs(g, co, k)
    fake["lib"].max_degree, fake["lib"].nonfinite = None, True
    xy = co.copy()
    sat = _expected(g, co, k)[0]
    xy[sat[3], 1] = np.nan  # a saturated node's coordinate, compared with every orphan
    with pytest.raises(ValueError) as host:
        _expected(g, xy, k)
    with pytest.raises(ValueError) as dev:
        S.sepal_idxs(g, xy, k)
    assert str(dev.value) == str(host.value) and "NaN" in str(dev.value)


def test_sepal_checks_keep_their_order(fake, case):
    import pandas as pd

    import squidpy_b200 as sq
    from squidpy_b200 import AnnDataLite

    g, co, k = case
    ad = AnnDataLite(X=np.ones((g.shape[0], 2)), obsp={"spatial_connectivities": g}, obsm={"spatial": co}, var=pd.DataFrame(index=["a", "b"]))
    with pytest.raises(ValueError, match="either `4` or `6`"):
        sq.gr.sepal(ad, max_neighs=5)
    with pytest.raises(ValueError, match="No genes"):
        sq.gr.sepal(ad, max_neighs=6, genes=[])
    with pytest.raises(ValueError, match=r"Expected `max_neighs=6`, found node with `4` neighbors"):
        sq.gr.sepal(ad, max_neighs=6)
    assert fake["lib"].calls and not fake["lib"].calls[0]["device_input"]


# --- the orphan rules ------------------------------------------------------------------------------------------------------


def _orphan_case(rng, n_sat=40, n_orph=12):
    """Integer-valued coordinates on a small range: many L1 ties."""
    return rng.integers(-4, 5, (n_orph, 2)).astype(np.float64), rng.integers(-4, 5, (n_sat, 2)).astype(np.float64)


def test_restatement_ties_follow_sklearn_argmin():
    rng = np.random.default_rng(0)
    for _ in range(20):
        o, s = _orphan_case(rng)
        n_s = len(s)
        # a graph whose saturated nodes are the ring 0..n_s-1 closed with k = 2, the orphans isolated
        ring = sp.csr_matrix((np.ones(2 * n_s), np.c_[(np.arange(n_s) - 1) % n_s, (np.arange(n_s) + 1) % n_s].ravel(), 2 * np.arange(n_s + 1)),
                             shape=(n_s, n_s))
        g = sp.block_diag([ring, sp.csr_matrix((len(o), len(o)))], format="csr")
        sat, _, unsat, unsat_idx = S._compute_idxs(g, np.r_[s, o], 2)
        assert np.array_equal(sat, np.arange(n_s))
        assert np.array_equal(unsat_idx, sat[pairwise_distances(o, s, metric="l1").argmin(1)])


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_restatement_refuses_non_finite_coordinates_as_sklearn(bad):
    rng = np.random.default_rng(1)
    o, s = _orphan_case(rng)
    s[5, 0] = bad
    with pytest.raises(ValueError) as ours:
        n_s = len(s)
        ring = sp.csr_matrix((np.ones(2 * n_s), np.c_[(np.arange(n_s) - 1) % n_s, (np.arange(n_s) + 1) % n_s].ravel(), 2 * np.arange(n_s + 1)),
                             shape=(n_s, n_s))
        S._compute_idxs(sp.block_diag([ring, sp.csr_matrix((len(o), len(o)))], format="csr"), np.r_[s, o], 2)
    with pytest.raises(ValueError) as theirs:
        pairwise_distances(o, s, metric="l1")
    assert str(ours.value) == str(theirs.value)


def _device_argmin(o, s, chunks):
    """The reduction of si_nearest / si_finish: key 0 for NaN, else the distance's bits + 1, the least (key, j) per chunk of the
    saturated nodes, then over the chunks."""
    with np.errstate(invalid="ignore"):  # inf - inf
        d = np.abs(o[:, None, 0] - s[None, :, 0]) + np.abs(o[:, None, 1] - s[None, :, 1])
    key = np.where(np.isnan(d), 0, d.view(np.uint64) + np.uint64(1))
    best = []
    for lo, hi in zip(chunks[:-1], chunks[1:]):
        if hi > lo:
            kk = key[:, lo:hi]
            j = kk.argmin(1)  # the first least key of the chunk
            best.append((kk[np.arange(len(o)), j], j + lo))
    return np.array([min((int(k[r]), int(j[r])) for k, j in best)[1] for r in range(len(o))])


def test_device_reduction_is_numpy_argmin_with_nan_and_inf():
    rng = np.random.default_rng(2)
    for t in range(30):
        o, s = _orphan_case(rng, n_sat=70, n_orph=15)
        if t % 3:
            s[rng.integers(0, len(s), 3), rng.integers(0, 2, 3)] = rng.choice([np.nan, np.inf, -np.inf], 3)
            o[rng.integers(0, len(o), 2), rng.integers(0, 2, 2)] = rng.choice([np.nan, np.inf, -np.inf], 2)
        want = np.argmin(cdist(o, s, "cityblock"), axis=1)
        for chunks in ([0, len(s)], [0, 7, 30, 31, len(s)], list(range(0, len(s) + 1, 9)) + [len(s)]):
            assert np.array_equal(_device_argmin(o, s, chunks), want)
