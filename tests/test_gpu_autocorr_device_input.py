"""spatial_autocorr on feature matrices resident in device memory: the DataFrame equals, bit for bit, the one computed from
the same matrix on the host (both paths end in the same device layout and run the same kernels), for every supported
format, dtype and gene selection; the caller's producer stream is honoured; invalid input raises like on the host and
leaves the context usable.  cupy is not needed: a cupy-like duck type wraps torch CUDA tensors."""

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
    """cupy-like dense device array: a torch CUDA tensor behind a version-3 interface (optionally naming its stream)."""

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
        raise AssertionError("a device matrix was read on the host")


class CuSparse:
    """cupyx.scipy.sparse-like CSR / CSC matrix made of torch CUDA tensors."""

    def __init__(self, fmt, indptr, indices, data, shape, stream=None):
        self.format, self.shape = fmt, tuple(shape)
        self.indptr, self.indices, self.data = (CuArray(torch.as_tensor(a).cuda(), stream) for a in (indptr, indices, data))

    @classmethod
    def of(cls, m, ip=np.int32, ix=np.int32, dt=None):
        return cls(m.format, m.indptr.astype(ip), m.indices.astype(ix), m.data if dt is None else m.data.astype(dt), m.shape)

    def __array__(self, *a, **k):
        raise AssertionError("a device matrix was read on the host")


def _w(r=30, c=40):
    g = synth.hex_graph(r, c)
    return sp.csr_matrix(g, dtype=np.float32)


def _adata(X, w, n_var, **kw):
    var = pd.DataFrame(index=[f"g{i}" for i in range(n_var)])
    return AnnDataLite(X=X, obsp={KEY: w}, var=var, shape=(w.shape[0], n_var), **kw)


def _x(n, g=37, density=0.15, seed=0, dtype=np.float32):
    x = sp.random(n, g, density=density, format="csr", random_state=seed, dtype=np.float64)
    x.data = np.round(x.data * 16) / 4
    x[:, 5] = 0.0  # an all-zero feature -> NaN scores
    x.eliminate_zeros()
    return x.astype(dtype)


def _same(a: pd.DataFrame, b: pd.DataFrame):
    assert list(a.columns) == list(b.columns)
    assert list(a.index) == list(b.index)
    assert np.array_equal(a.to_numpy(np.float64), b.to_numpy(np.float64), equal_nan=True)


def _both(x_host, x_dev, w, n_var, modes=("moran", "geary"), **kw):
    for mode in modes:
        host = sq.gr.spatial_autocorr(_adata(x_host, w, n_var), mode=mode, copy=True, **kw)
        dev = sq.gr.spatial_autocorr(_adata(x_dev, w, n_var), mode=mode, copy=True, **kw)
        _same(dev, host)


@pytest.mark.parametrize("case", ["csr32", "csr64", "csr_mixed", "torch_csr", "csc", "torch_csc", "unsorted"])
def test_sparse_formats(case):
    w = _w()
    x = _x(w.shape[0])
    if case == "csr32":
        dev = CuSparse.of(x)
    elif case == "csr64":
        dev = CuSparse.of(x, np.int64, np.int64)
    elif case == "csr_mixed":
        dev = CuSparse.of(x, np.int64, np.int32)
    elif case == "torch_csr":
        dev = torch.sparse_csr_tensor(torch.from_numpy(x.indptr.astype(np.int64)), torch.from_numpy(x.indices.astype(np.int64)),
                                      torch.from_numpy(x.data), size=x.shape).cuda()
    elif case == "csc":
        x = x.tocsc()
        dev = CuSparse.of(x)
    elif case == "torch_csc":
        x = x.tocsc()
        dev = torch.sparse_csc_tensor(torch.from_numpy(x.indptr.astype(np.int64)), torch.from_numpy(x.indices.astype(np.int64)),
                                      torch.from_numpy(x.data), size=x.shape).cuda()
    else:
        rng = np.random.default_rng(1)
        x = x.copy()
        for r in range(x.shape[0]):  # every row's entries in a random order
            a, b = x.indptr[r], x.indptr[r + 1]
            p = rng.permutation(b - a)
            x.indices[a:b], x.data[a:b] = x.indices[a:b][p], x.data[a:b][p]
        x.has_sorted_indices = False
        dev = CuSparse.of(x)
    _both(x, dev, w, x.shape[1])


@pytest.mark.parametrize("order", ["C", "F", "strided"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_dense_layouts(order, dtype):
    w = _w()
    x = _x(w.shape[0], dtype=dtype).toarray()
    if order == "C":
        t = torch.from_numpy(x).cuda()
    elif order == "F":
        t = torch.from_numpy(x).cuda().t().contiguous().t()
    else:
        wide = np.repeat(x, 2, axis=1)
        wide[:, 1::2] = -7.0
        t = torch.from_numpy(wide).cuda()[:, ::2]
        assert not t.is_contiguous()
    _both(x, CuArray(t), w, x.shape[1])


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.int32])
@pytest.mark.parametrize("kind", ["sparse", "dense"])
def test_data_dtypes(dtype, kind):
    w = _w()
    x = _x(w.shape[0], dtype=np.float64)
    data = x.data.astype(dtype)
    if kind == "sparse":
        dev = CuSparse(x.format, x.indptr, x.indices, data, x.shape)
        # scipy has no float16 matrices: the host twin holds the float16 values as float64 (the host path's conversion)
        host = sp.csr_matrix((data.astype(np.float64) if dtype == np.float16 else data, x.indices, x.indptr), shape=x.shape)
    else:
        dense = x.toarray().astype(dtype)
        dev, host = CuArray(torch.from_numpy(dense).cuda()), dense
    _both(host, dev, w, x.shape[1])


def test_gene_selection():
    w = _w()
    n = w.shape[0]
    x = _x(n, g=30)
    dev = CuSparse.of(x)
    rng = np.random.default_rng(4)
    names = [f"g{i}" for i in range(30)]
    _both(x, dev, w, 30, genes=list(rng.permutation(names)[:11]))  # shuffled subset
    _both(x, dev, w, 30, genes=["g3", "g9", "g3", "g0", "g9"], modes=("moran",))  # duplicates: scored once, expanded
    _both(x, dev, w, 30, genes="g7", modes=("geary",))
    # the highly_variable default
    hv = np.zeros(30, bool)
    hv[[1, 4, 8, 20, 29]] = True
    for X in (x, dev):
        a = _adata(X, w, 30)
        a.var["highly_variable"] = hv
        if X is x:
            host = sq.gr.spatial_autocorr(a, copy=True)
        else:
            _same(sq.gr.spatial_autocorr(a, copy=True), host)
    # layer=
    host = sq.gr.spatial_autocorr(_adata(None, w, 30, layers={"counts": x}), layer="counts", genes=names[:9], copy=True)
    _same(sq.gr.spatial_autocorr(_adata(None, w, 30, layers={"counts": dev}), layer="counts", genes=names[:9], copy=True), host)


def test_use_raw_and_obsm():
    w = _w()
    n = w.shape[0]
    x, raw_x = _x(n, g=20, seed=1), _x(n, g=26, seed=2)
    raw_var = pd.DataFrame(index=[f"g{i}" for i in range(26)][::-1])  # raw has more variables, in another order
    genes = ["g2", "g19", "g7", "g0", "g25"]  # g25 exists in raw only
    host = _adata(x, w, 20, raw=AnnDataLite(X=raw_x, var=raw_var))
    dev = _adata(CuSparse.of(x), w, 20, raw=AnnDataLite(X=CuSparse.of(raw_x), var=raw_var))
    for mode in ("moran", "geary"):
        _same(sq.gr.spatial_autocorr(dev, use_raw=True, genes=genes, mode=mode, copy=True),
              sq.gr.spatial_autocorr(host, use_raw=True, genes=genes, mode=mode, copy=True))
    emb = np.random.default_rng(3).standard_normal((n, 8)).astype(np.float32)
    host.obsm["emb"], dev.obsm["emb"] = emb, CuArray(torch.from_numpy(emb).cuda())
    for genes in (None, [5, 1, 6]):
        _same(sq.gr.spatial_autocorr(dev, attr="obsm", layer="emb", genes=genes, copy=True),
              sq.gr.spatial_autocorr(host, attr="obsm", layer="emb", genes=genes, copy=True))


def test_all_zero_matrix():
    w = _w()
    x = sp.csr_matrix((w.shape[0], 9), dtype=np.float32)
    _both(x, CuSparse(x.format, x.indptr, x.indices.astype(np.int32), x.data, x.shape), w, 9)


def test_million_observations_global_bitmap():
    """1M observations: the per-feature bitmap lives in global memory; X is built on the device."""
    w = sp.csr_matrix(synth.hex_graph(1000, 1000), dtype=np.float32)
    n = w.shape[0]
    gen = torch.Generator(device="cuda").manual_seed(5)
    dense = torch.rand((n, 6), device="cuda", generator=gen)
    dense = torch.where(dense < 0.05, torch.round(dense * 400), torch.zeros_like(dense))
    dev = dense.to_sparse_csr()
    host = sp.csr_matrix((dev.values().cpu().numpy(), dev.col_indices().cpu().numpy(), dev.crow_indices().cpu().numpy()), shape=(n, 6))
    _both(host, dev, w, 6)


def test_permutations_match_host():
    w = _w()
    x = _x(w.shape[0], g=12)
    for mode in ("moran", "geary"):
        host = sq.gr.spatial_autocorr(_adata(x, w, 12), mode=mode, n_perms=40, seed=11, copy=True, genes=["g1", "g4", "g1", "g9"])
        dev = sq.gr.spatial_autocorr(_adata(CuSparse.of(x), w, 12), mode=mode, n_perms=40, seed=11, copy=True, genes=["g1", "g4", "g1", "g9"])
        assert "pval_sim" in dev.columns
        _same(dev, host)


def test_device_weight_matrix_is_copied_to_host():
    w = _w()
    x = _x(w.shape[0])
    wd = torch.sparse_csr_tensor(torch.from_numpy(w.indptr.astype(np.int64)), torch.from_numpy(w.indices.astype(np.int64)),
                                 torch.from_numpy(w.data), size=w.shape).cuda()
    a = _adata(CuSparse.of(x), w, x.shape[1])
    b = _adata(CuSparse.of(x), wd, x.shape[1])
    _same(sq.gr.spatial_autocorr(b, copy=True), sq.gr.spatial_autocorr(a, copy=True))


def test_producer_stream_is_waited_for():
    """X is written on a side stream behind a long sleep; the library must wait for it through the interface's stream."""
    w = _w()
    x = _x(w.shape[0])
    dense = x.toarray()
    src_dense = torch.from_numpy(dense).cuda()
    src_data = torch.from_numpy(x.data).cuda()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t_dense = torch.zeros_like(src_dense)
        t_data = torch.zeros_like(src_data)
        torch.cuda._sleep(200_000_000)
        t_dense.add_(src_dense)
        t_data.add_(src_data)
    s = side.cuda_stream
    sparse = CuSparse(x.format, x.indptr, x.indices, np.zeros(0), x.shape, stream=s)
    sparse.data = CuArray(t_data, s)
    for X, H in ((CuArray(t_dense, s), dense), (sparse, x)):
        got = sq.gr.spatial_autocorr(_adata(X, w, x.shape[1]), copy=True)
        _same(got, sq.gr.spatial_autocorr(_adata(H, w, x.shape[1]), copy=True))
    torch.cuda.synchronize()
    assert torch.equal(t_dense, src_dense) and torch.equal(t_data, src_data)  # the caller's buffers are untouched


def _corrupt(x, **arrays):
    """A host CSR whose arrays are replaced without scipy's validation, and its device twin."""
    h = x.copy()
    for k, v in arrays.items():
        setattr(h, k, np.asarray(v, dtype=getattr(h, k).dtype))
    return h, CuSparse(h.format, h.indptr, h.indices, h.data, h.shape)


def test_invalid_input_raises_like_the_host_and_context_survives():
    w = _w()
    n = w.shape[0]
    x = _x(n, g=10, density=0.3)
    good = CuSparse.of(x)
    ok = sq.gr.spatial_autocorr(_adata(good, w, 10), copy=True)
    r = int(np.flatnonzero(np.diff(x.indptr) >= 2)[0])
    a = x.indptr[r]
    dup = x.indices.copy()
    dup[a + 1] = dup[a]
    oor = x.indices.copy()
    oor[a] = 10
    dec = x.indptr.copy()
    dec[r + 1] = dec[r] - 1 if dec[r] > 0 else dec[r + 2] + 1
    for arrays, match in (({"indices": dup}, "stored twice"), ({"indices": oor}, "out of range"), ({"indptr": dec}, "indptr")):
        h, d = _corrupt(x, **arrays)
        with pytest.raises(Exception) as host_err:
            sq.gr.spatial_autocorr(_adata(h, w, 10), copy=True)
        with pytest.raises(type(host_err.value), match=match):
            sq.gr.spatial_autocorr(_adata(d, w, 10), copy=True)
        _same(sq.gr.spatial_autocorr(_adata(good, w, 10), copy=True), ok)
    with pytest.raises(ValueError, match="does not match"):
        sq.gr.spatial_autocorr(_adata(good, w, 10), device=torch.cuda.device_count(), copy=True)
    host_mem = np.zeros((n, 10), np.float32)

    class HostCAI:
        shape = host_mem.shape
        __cuda_array_interface__ = {"shape": host_mem.shape, "typestr": "<f4", "data": (host_mem.ctypes.data, False), "version": 3,
                                    "strides": None, "stream": None}

    with pytest.raises(ValueError, match="host memory"):
        sq.gr.spatial_autocorr(_adata(HostCAI(), w, 10), copy=True)
    coo = torch.sparse_coo_tensor(torch.tensor([[0, 1], [2, 3]]), torch.tensor([1.0, 2.0]), size=(n, 10)).cuda()
    with pytest.raises(NotImplementedError, match="csr, csc"):
        sq.gr.spatial_autocorr(_adata(coo, w, 10), copy=True)
    _same(sq.gr.spatial_autocorr(_adata(good, w, 10), copy=True), ok)
