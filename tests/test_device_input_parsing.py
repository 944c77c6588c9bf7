"""Host logic of device-resident input (no GPU, no library call): CUDA Array Interface parsing, format detection, the
feature map that expresses gene subsets, duplicates and shards, and the guarantee that X is never read on the host."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

from squidpy_b200._device import DevArray, DevSparse, array_device, common_stream, device_matrix, dtype_code, feature_map, parse_cai
from squidpy_b200._dist import shard_range


class FakeDev:
    """An object exposing a hand-written __cuda_array_interface__; reading it on the host fails."""

    def __init__(self, shape, typestr="<f4", strides=None, ptr=0x7000_0000, version=3, stream=None, **extra):
        self.shape = tuple(shape)
        self.__cuda_array_interface__ = dict(shape=self.shape, typestr=typestr, data=(ptr, False), strides=strides, version=version,
                                             stream=stream, **extra)

    def __array__(self, *a, **k):
        raise AssertionError("__array__ called on a device array")


class FakeSparse:
    def __init__(self, fmt, shape, n_ptr=5, nnz=7, stream=None):
        self.format, self.shape = fmt, shape
        self.indptr = FakeDev((n_ptr,), "<i8", ptr=0x1000, stream=stream)
        self.indices = FakeDev((nnz,), "<i4", ptr=0x2000, stream=stream)
        self.data = FakeDev((nnz,), "<f8", ptr=0x3000, stream=stream)

    def __array__(self, *a, **k):
        raise AssertionError("__array__ called on a device matrix")


def test_cai_typestr_strides_version_stream():
    a = parse_cai(FakeDev((4, 6)))
    assert a.dtype == np.float32 and a.shape == (4, 6) and a.strides == (6, 1) and a.stream == 0 and a.ptr == 0x7000_0000
    f = parse_cai(FakeDev((4, 6), "<f8", strides=(8, 32)))  # F order, byte strides -> element strides
    assert f.dtype == np.float64 and f.strides == (1, 4)
    v = parse_cai(FakeDev((10, 3), "<f2", strides=(12, 4)))  # X[:, ::2] of a (10, 6) float16 array
    assert v.strides == (6, 2) and dtype_code(v) == 2
    assert parse_cai(FakeDev((3,), "<i8", stream=1)).stream == 1
    assert parse_cai(FakeDev((3,), "<i8", stream=12345)).stream == 12345
    assert parse_cai(FakeDev((3,), "<i8", version=2, stream=99)).stream == 0  # `stream` is a version-3 field
    assert parse_cai(FakeDev((3,), "<i8", stream=7), stream=4).stream == 4
    assert [dtype_code(parse_cai(FakeDev((1,), t))) for t in ("<f4", "<f8", "<f2", "<i4", "<i8")] == [0, 1, 2, 3, 4]


@pytest.mark.parametrize(
    "kw, exc, match",
    [
        (dict(mask=(1, False)), ValueError, "Masked"),
        (dict(version=9), ValueError, "version"),
        (dict(stream=0), ValueError, "ambiguous"),
        (dict(typestr=">f4"), ValueError, "Big-endian"),
        (dict(strides=(6, 3)), ValueError, "multiples"),
    ],
)
def test_cai_rejections(kw, exc, match):
    with pytest.raises(exc, match=match):
        parse_cai(FakeDev((4, 6), **kw))


def test_unsupported_dtype():
    with pytest.raises(TypeError, match="uint8"):
        dtype_code(parse_cai(FakeDev((2,), "|u1")))


def test_format_detection():
    assert device_matrix(np.zeros((2, 2))) is None
    assert device_matrix(sp.random(4, 4, density=0.5, format="csr")) is None
    assert device_matrix(sp.random(4, 4, density=0.5, format="coo")) is None
    assert isinstance(device_matrix(FakeDev((4, 2))), DevArray)
    d = device_matrix(FakeSparse("csr", (4, 9)))
    assert isinstance(d, DevSparse) and d.format == "csr" and d.shape == (4, 9)
    assert d.indptr.dtype == np.int64 and d.indices.dtype == np.int32 and d.data.dtype == np.float64
    assert device_matrix(FakeSparse("csc", (4, 9), n_ptr=10)).format == "csc"
    for fmt in ("coo", "bsr", "dia"):
        with pytest.raises(NotImplementedError, match="csr, csc"):
            device_matrix(FakeSparse(fmt, (4, 9)))


def test_torch_layouts_without_gpu():
    torch = pytest.importorskip("torch")
    t = torch.zeros((3, 2))
    assert device_matrix(t) is None  # a CPU tensor takes the host path
    assert device_matrix(t.to_sparse_csr()) is None
    with pytest.raises(NotImplementedError, match="csr, csc"):
        device_matrix(t.to_sparse())  # COO


def test_streams_and_devices():
    assert common_stream(device_matrix(FakeSparse("csr", (4, 9), stream=5))) == 5
    s = FakeSparse("csr", (4, 9))
    s.data = FakeDev((7,), "<f8", ptr=0x3000, stream=6)
    assert common_stream(device_matrix(s)) == 6
    s.indptr = FakeDev((5,), "<i8", ptr=0x1000, stream=8)
    with pytest.raises(ValueError, match="different producer streams"):
        common_stream(device_matrix(s))
    d = device_matrix(FakeSparse("csr", (4, 9)))
    assert array_device(d, lambda p: 1) == 1
    with pytest.raises(ValueError, match="host memory"):
        array_device(d, lambda p: -1)
    with pytest.raises(ValueError, match="different devices"):
        array_device(d, lambda p: 0 if p == 0x1000 else 1)
    empty = FakeSparse("csr", (4, 9), nnz=0)
    empty.indices = FakeDev((0,), "<i4", ptr=0)
    empty.data = FakeDev((0,), "<f8", ptr=0)
    seen = []
    assert array_device(device_matrix(empty), lambda p: seen.append(p) or 0) == 0 and seen == [0x1000]


def test_feature_map_subsets_and_duplicates():
    cm, n_out, expand = feature_map(10, [7, 2, 5])
    assert n_out == 3 and cm.dtype == np.int32 and list(cm) == [-1, -1, 1, -1, -1, 2, -1, 0, -1, -1] and list(expand) == [0, 1, 2]
    cm, n_out, expand = feature_map(6, [4, 1, 4, 0, 1])  # duplicates are loaded once, in order of first occurrence
    assert n_out == 3 and list(cm) == [2, 1, -1, -1, 0, -1] and list(expand) == [0, 1, 0, 2, 1]
    scores = np.array([40.0, 10.0, 0.0])  # loaded features 4, 1, 0
    assert list(scores[expand]) == [40.0, 10.0, 40.0, 0.0, 10.0]
    with pytest.raises(IndexError):
        feature_map(3, [0, 3])


@pytest.mark.parametrize("ws", [2, 3])
def test_feature_map_shards_cover_the_selection_once(ws):
    rng = np.random.default_rng(ws)
    sel = rng.integers(0, 40, 23)  # with repeats
    parts = []
    for rank in range(ws):
        lo, hi = shard_range(len(sel), rank, ws)
        cm, n_out, expand = feature_map(40, sel, lo, hi)
        loaded = np.full(n_out, -1)
        loaded[cm[cm >= 0]] = np.flatnonzero(cm >= 0)  # output index -> input feature
        assert (cm >= 0).sum() == n_out and sorted(cm[cm >= 0]) == list(range(n_out))
        parts.append(loaded[expand])
    assert np.array_equal(np.concatenate(parts), sel)


def test_use_raw_gene_order_and_no_host_read(monkeypatch):
    """The device path resolves genes from var / raw.var_names with the host path's code and never touches X on the host;
    the library is replaced by a recorder."""
    import squidpy_b200.gr._ppatterns as pp
    from squidpy_b200 import AnnDataLite

    n = 12
    w = sp.csr_matrix(np.eye(n, k=1) + np.eye(n, k=-1), dtype=np.float32)
    raw_var = pd.DataFrame(index=[f"r{i}" for i in range(8)])
    X = FakeDev((n, 5))
    adata = AnnDataLite(X=X, obsp={"spatial_connectivities": w}, var=pd.DataFrame(index=[f"r{i}" for i in range(5)]),
                        raw=AnnDataLite(X=FakeDev((n, 8)), var=raw_var))
    seen = {}

    class Plan:
        def __init__(self, g, ctx):
            self.n = g.shape[0]

        def load(self, m, *, obs_major, col_map):
            seen["m"], seen["col_map"] = m, col_map
            self.k = int(col_map.max()) + 1

        def score(self, mode):
            return np.arange(self.k, dtype=np.float64)

        def close(self):
            pass

    class Ctx:
        device = 0

        import threading

        lock = threading.RLock()

    monkeypatch.setattr(pp, "AutocorrPlan", Plan)
    monkeypatch.setattr(pp, "default_context", lambda device=None: Ctx())
    monkeypatch.setattr(pp, "pointer_device", lambda p: 0)
    genes = ["r6", "r2", "r9", "r0"]  # r9 is not in raw
    df = pp.spatial_autocorr(adata, genes=genes, use_raw=True, copy=True)
    expected = list(set(genes) & set(raw_var.index))  # the host path's (set-ordered) list
    assert seen["m"] is adata.raw.X and sorted(df.index) == sorted(expected)
    cm = seen["col_map"]
    order = [raw_var.index.get_loc(g) for g in expected]
    assert list(np.flatnonzero(cm >= 0)) == sorted(order) and [cm[i] for i in order] == list(range(len(order)))
    # scores come back in the list's order: score k belongs to expected[k]
    assert dict(zip(df.index, df["I"])) == {g: float(k) for k, g in enumerate(expected)}
