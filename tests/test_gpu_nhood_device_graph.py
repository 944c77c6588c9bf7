"""nhood_enrichment and interaction_matrix on neighbour graphs resident in GPU memory: with the same seed the results equal,
bit for bit, those computed from the same graph on the host (both paths end in the same uint32 CSR on the device, or the same
kernel), for every accepted format, index width and value dtype; the caller's producer stream is honoured; invalid graphs
raise like on the host and leave the context usable.  cupy is not needed: a cupy-like duck type wraps torch CUDA tensors,
and reading it on the host fails the test."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu
KEY = "spatial_connectivities"


class CuArray:
    """cupy-like device array: a torch CUDA tensor behind a version-3 interface (optionally naming its stream)."""

    def __init__(self, t, stream=None):
        self.t, self.stream = t, stream

    @property
    def shape(self):
        return tuple(self.t.shape)

    @property
    def __cuda_array_interface__(self):
        d = dict(self.t.__cuda_array_interface__)
        d.update(version=3, stream=self.stream)
        return d

    def __array__(self, *a, **k):
        raise AssertionError("a device graph was read on the host")


class CuSparse:
    """cupyx.scipy.sparse-like CSR / CSC matrix made of torch CUDA tensors."""

    def __init__(self, fmt, indptr, indices, data, shape, stream=None):
        self.format, self.shape = fmt, tuple(shape)
        self.indptr, self.indices, self.data = (CuArray(torch.as_tensor(a).cuda(), stream) for a in (indptr, indices, data))

    @classmethod
    def of(cls, m, ip=np.int32, ix=np.int32):
        return cls(m.format, m.indptr.astype(ip), m.indices.astype(ix), m.data, m.shape)

    def __array__(self, *a, **k):
        raise AssertionError("a device graph was read on the host")


def _torch_sparse(m):
    ip, ix, v = (torch.from_numpy(np.asarray(a)) for a in (m.indptr.astype(np.int64), m.indices.astype(np.int64), m.data))
    make = torch.sparse_csr_tensor if m.format == "csr" else torch.sparse_csc_tensor
    return make(ip, ix, v, size=m.shape).cuda()


FORMATS = ["csr32", "csr64", "csr_mixed", "csc", "csc64", "torch_csr", "torch_csc"]


def _formats(g, fmt):
    """(host graph, device graph) of the CSR ``g`` in format ``fmt``; the host twin of a CSC graph is scipy CSC."""
    if fmt.startswith("csc") or fmt == "torch_csc":
        g = g.tocsc()
    if fmt in ("torch_csr", "torch_csc"):
        return g, _torch_sparse(g)
    ip, ix = {"csr32": (np.int32, np.int32), "csr64": (np.int64, np.int64), "csr_mixed": (np.int64, np.int32), "csc": (np.int32, np.int32),
              "csc64": (np.int64, np.int32)}[fmt]
    return g, CuSparse.of(g, ip, ix)


def _raw(indptr, indices, n, data=None):
    """A scipy CSR holding exactly these arrays (duplicates, unsorted rows and explicit zeros kept)."""
    indices = np.asarray(indices, np.int32)
    data = np.ones(indices.size, np.float32) if data is None else data
    return sp.csr_matrix((data, indices, np.asarray(indptr, np.int32)), shape=(n, n))


def _graph(kind):
    if kind == "hex":  # structurally symmetric: row records of the upper triangle + mirrored flush
        return synth.hex_graph(30, 40)
    if kind == "knn":  # directed kNN: records of every entry
        return synth.knn_graph(synth.hex_coords(30, 40) + np.random.default_rng(0).normal(0, 7, (1200, 2)), k=6)
    if kind == "self_loops":
        g = synth.hex_graph(30, 40) + sp.eye(1200, dtype=np.float32, format="csr")
        return g.tocsr()
    if kind == "messy":  # duplicate and unsorted column indices, stored explicit zeros
        g = synth.hex_graph(30, 40)
        rng = np.random.default_rng(2)
        idx, data, ptr = [], [], [0]
        for r in range(g.shape[0]):
            row = list(g.indices[g.indptr[r] : g.indptr[r + 1]])
            if r % 3 == 0:
                row.append(row[0])
            rng.shuffle(row)
            idx += row
            data += [0.0 if r % 5 == 0 else 1.0] * len(row)
            ptr.append(len(idx))
        return _raw(ptr, idx, g.shape[0], np.asarray(data, np.float32))
    if kind == "empty_rows":
        g = synth.hex_graph(30, 40).tolil()
        g[::7] = 0  # every 7th row empty
        g = g.tocsr()
        g.eliminate_zeros()
        return g
    assert kind == "nnz0"
    return sp.csr_matrix((1200, 1200), dtype=np.float32)


def _adata(g, n, n_cls, seed=0, libs=None, nan=False):
    codes = np.random.default_rng(seed).integers(0, n_cls, n)
    if nan:
        codes[::11] = -1
    obs = pd.DataFrame({"cl": pd.Categorical.from_codes(codes, categories=[f"c{i:03d}" for i in range(n_cls)])}, index=[str(i) for i in range(n)])
    if libs is not None:
        obs["lib"] = pd.Categorical.from_codes(np.arange(n) * libs // n, categories=[f"L{i}" for i in range(libs)])
    return AnnDataLite(obs=obs, obsp={KEY: g}, shape=(n, 1))


def _nhood_same(host, dev, n_cls=3, n_perms=24, seed=7, libs=None, **kw):
    n = host.shape[0]
    h = sq.gr.nhood_enrichment(_adata(host, n, n_cls, libs=libs), "cl", library_key="lib" if libs else None, n_perms=n_perms, seed=seed,
                               copy=True, **kw)
    d = sq.gr.nhood_enrichment(_adata(dev, n, n_cls, libs=libs), "cl", library_key="lib" if libs else None, n_perms=n_perms, seed=seed,
                               copy=True, **kw)
    assert d.counts.dtype == h.counts.dtype and d.zscore.dtype == h.zscore.dtype
    assert np.array_equal(d.counts, h.counts)
    assert np.array_equal(d.zscore, h.zscore, equal_nan=True)
    return h


@pytest.mark.parametrize("n_cls", [2, 300])  # 300: more than 256 clusters, 16-bit labels
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("kind", ["hex", "knn", "self_loops", "messy", "empty_rows", "nnz0"])
def test_nhood_matches_host(kind, fmt, n_cls):
    host, dev = _formats(_graph(kind), fmt)
    res = _nhood_same(host, dev, n_cls=n_cls, n_perms=12 if n_cls > 256 else 24)
    if kind != "nnz0":
        assert res.counts.sum() > 0


@pytest.mark.parametrize("rng", ["numpy", "philox"])
@pytest.mark.parametrize("fmt", ["csr32", "csc", "torch_csr"])
def test_nhood_library_key_and_rng(fmt, rng):
    host, dev = _formats(_graph("knn"), fmt)
    _nhood_same(host, dev, n_cls=5, n_perms=40, libs=3, rng=rng)
    _nhood_same(host, dev, n_cls=5, n_perms=40, rng=rng)


@pytest.mark.parametrize("fmt", ["csr_mixed", "torch_csc"])
def test_nhood_region_replay_size(fmt):
    """>= 512 K spots and more permutations than twice the SM count: the exact mode takes the region replay."""
    g = synth.hex_graph(725, 725)
    n_perms = 2 * sq.default_context(0).sm_count + 8
    assert g.shape[0] >= 524_288 and n_perms > 2 * sq.default_context(0).sm_count
    host, dev = _formats(g, fmt)
    _nhood_same(host, dev, n_cls=12, n_perms=n_perms, seed=3)


# ---- interaction_matrix -----------------------------------------------------------------------------------------------
def _inter(g, n_cls=6, nan=True, **kw):
    return sq.gr.interaction_matrix(_adata(g, g.shape[0], n_cls, seed=4, nan=nan), "cl", copy=True, **kw)


@pytest.mark.parametrize("normalized", [False, True])
@pytest.mark.parametrize("weights", [False, True])
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("kind", ["knn", "messy", "nnz0"])
def test_interaction_matches_host(kind, fmt, weights, normalized):
    g = _graph(kind)
    g.data = np.random.default_rng(5).integers(0, 4, g.nnz).astype(np.float32)  # integer-valued: every path sums exactly
    host, dev = _formats(g, fmt)
    for nan in (False, True):
        h = _inter(host, nan=nan, weights=weights, normalized=normalized)
        d = _inter(dev, nan=nan, weights=weights, normalized=normalized)
        assert d.dtype == h.dtype
        assert np.array_equal(d, h, equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.int32, np.int64, bool])
@pytest.mark.parametrize("fmt", ["csr32", "csc", "torch_csr"])
def test_interaction_value_dtypes(dtype, fmt):
    g = _graph("knn")
    rng = np.random.default_rng(6)
    if np.dtype(dtype).kind == "f":
        vals = rng.random(g.nnz).astype(dtype)
    elif dtype is bool:
        vals = rng.random(g.nnz) < 0.7
    else:
        vals = rng.integers(-3, 9, g.nnz).astype(dtype)
    # scipy has no float16 matrices: the host twin holds the float16 values as float64 (the host path's conversion)
    host = sp.csr_matrix((vals.astype(np.float64) if dtype == np.float16 else vals, g.indices, g.indptr), shape=g.shape)
    if fmt == "torch_csr":
        dev = torch.sparse_csr_tensor(torch.from_numpy(g.indptr.astype(np.int64)), torch.from_numpy(g.indices.astype(np.int64)),
                                      torch.from_numpy(vals), size=g.shape).cuda()
    else:
        src = host.tocsc() if fmt == "csc" else host
        dev = CuSparse(src.format, src.indptr, src.indices, src.data.astype(dtype), src.shape)
    for weights in (False, True):
        h = _inter(host, weights=weights)
        d = _inter(dev, weights=weights)
        assert d.dtype == h.dtype == (np.int64 if np.dtype(dtype).kind in "biu" else np.float64)
        if weights and np.dtype(dtype).kind == "f":
            np.testing.assert_allclose(d, h, rtol=1e-12, atol=0)
        else:
            assert np.array_equal(d, h)


# ---- stream ordering --------------------------------------------------------------------------------------------------
def test_producer_stream_is_waited_for():
    """The graph is written on a side stream behind a long sleep; the library must wait for it (CAI v3 `stream`, and torch's
    current stream for torch tensors)."""
    g = _graph("knn")
    n = g.shape[0]
    src = [torch.from_numpy(a.astype(np.int64)).cuda() for a in (g.indptr, g.indices)]
    vals = torch.from_numpy(g.data).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        ip, ix = (torch.zeros_like(s) for s in src)
        torch.cuda._sleep(200_000_000)
        ip.add_(src[0])
        ix.add_(src[1])
    cai = CuSparse("csr", np.zeros(0), np.zeros(0), np.zeros(0), g.shape, stream=side.cuda_stream)
    cai.indptr, cai.indices, cai.data = CuArray(ip, side.cuda_stream), CuArray(ix, side.cuda_stream), CuArray(vals, side.cuda_stream)
    _nhood_same(g, cai)
    assert np.array_equal(_inter(cai), _inter(g))
    torch.cuda.synchronize()

    with torch.cuda.stream(side):  # a torch tensor written on torch's current stream
        ip2, ix2 = (torch.zeros_like(s) for s in src)
        torch.cuda._sleep(200_000_000)
        ip2.add_(src[0])
        ix2.add_(src[1])
        t = torch.sparse_csr_tensor(ip2, ix2, vals, size=(n, n))
        _nhood_same(g, t)
        assert np.array_equal(_inter(t, weights=True), _inter(g, weights=True))
    torch.cuda.synchronize()
    assert torch.equal(ip, src[0]) and torch.equal(ix2, src[1])  # the caller's buffers are untouched


# ---- invalid input ----------------------------------------------------------------------------------------------------
def _corrupt(g, ix_dtype=np.int32, **arrays):
    """A host CSR whose arrays are replaced without scipy's validation, and its device twin."""
    h = g.copy()
    h.indices = h.indices.astype(ix_dtype)
    for k, v in arrays.items():
        setattr(h, k, np.asarray(v, dtype=getattr(h, k).dtype))
    return h, CuSparse(h.format, h.indptr, h.indices, h.data, h.shape)


def _both_raise(h, d):
    """The device graph raises the host graph's exception type, in both functions."""
    for call in (lambda G: _nhood_same_one(G), lambda G: _inter(G)):
        with pytest.raises(Exception) as host_err:
            call(h)
        with pytest.raises(type(host_err.value)):
            call(d)


def _nhood_same_one(G):
    return sq.gr.nhood_enrichment(_adata(G, G.shape[0], 3), "cl", n_perms=8, seed=1, copy=True)


def test_invalid_graphs_raise_like_the_host_and_context_survives():
    g = _graph("knn")
    n = g.shape[0]
    good = CuSparse.of(g)
    ok_n, ok_i = _nhood_same_one(g), _inter(g)

    def still_ok():
        r = _nhood_same_one(good)
        assert np.array_equal(r.counts, ok_n.counts) and np.array_equal(r.zscore, ok_n.zscore, equal_nan=True)
        assert np.array_equal(_inter(good), ok_i)

    first = g.indptr.copy()
    first[0] = 1
    dec = g.indptr.copy()
    dec[11] = dec[10] - 1
    last = g.indptr.copy()
    last[-1] = g.nnz - 1
    big = g.indices.copy()
    big[17] = n
    neg = g.indices.copy()
    neg[23] = -1
    cases = [dict(indptr=first), dict(indptr=dec), dict(indptr=last), dict(indices=big), dict(indices=neg), dict(indices=neg, ix_dtype=np.int64)]
    for arrays in cases:
        h, d = _corrupt(g, **arrays)
        _both_raise(h, d)
        still_ok()
    # int64 indices beyond 2^32 must not wrap into range
    wrap = g.indices.astype(np.int64)
    wrap[5] += 1 << 32
    for call in (_nhood_same_one, _inter):
        with pytest.raises(ValueError):
            call(CuSparse("csr", g.indptr, wrap, g.data, g.shape))
    still_ok()
    # non-square graph, and a square graph of the wrong size
    for shape in ((n, n + 1), (n + 1, n + 1)):
        ip = np.concatenate([g.indptr, np.full(shape[0] - n, g.nnz, g.indptr.dtype)])
        bad = CuSparse("csr", ip, g.indices, g.data, shape)
        with pytest.raises(ValueError, match="shape"):
            _nhood_same_one_labels(bad, n)
        with pytest.raises(ValueError, match="shape"):
            sq.gr.interaction_matrix(_adata(bad, n, 3), "cl", copy=True)
    h = sp.csr_matrix((g.data, g.indices, np.concatenate([g.indptr, [g.nnz]])), shape=(n + 1, n + 1))
    with pytest.raises(ValueError):  # the host path refuses a graph of another size too
        _nhood_same_one_labels(h, n)
    still_ok()
    # device= naming another device than the graph's
    for call in (lambda: sq.gr.nhood_enrichment(_adata(good, n, 3), "cl", n_perms=4, device=torch.cuda.device_count(), copy=True),
                 lambda: sq.gr.interaction_matrix(_adata(good, n, 3), "cl", device=torch.cuda.device_count(), copy=True)):
        with pytest.raises(ValueError, match="does not match"):
            call()
    # host memory behind the interface
    host_ip, host_ix = g.indptr.astype(np.int32), g.indices.astype(np.int32)

    class HostCAI:
        def __init__(self, a, t):
            self.shape = a.shape
            self.__cuda_array_interface__ = {"shape": a.shape, "typestr": t, "data": (a.ctypes.data, False), "version": 3, "strides": None,
                                             "stream": None}

    class HostSparse:
        format, shape = "csr", g.shape
        indptr, indices, data = HostCAI(host_ip, "<i4"), HostCAI(host_ix, "<i4"), HostCAI(g.data, "<f4")

    for call in (_nhood_same_one, _inter):
        with pytest.raises(ValueError, match="host memory"):
            call(HostSparse())
    # a dense device graph
    dense = torch.from_numpy(g.toarray()).cuda()
    for call in (_nhood_same_one, _inter):
        with pytest.raises(NotImplementedError, match="csr, csc"):
            call(dense)
    still_ok()


def _nhood_same_one_labels(G, n):
    return sq.gr.nhood_enrichment(_adata(G, n, 3), "cl", n_perms=8, seed=1, copy=True)
