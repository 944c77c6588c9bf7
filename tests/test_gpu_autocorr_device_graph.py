"""spatial_autocorr on weight matrices resident in GPU memory: a device CSR with float32 / float64 values and canonical rows is
row-normalised, summed and reduced to its moments on the device, and the DataFrame equals, bit for bit, the one computed from
the same graph on the host, in every column and in row order.  The caller's graph is never read on the host or modified.
Every other device graph (CSC, integer / bool values, unsorted or repeated columns) takes the host copy and still equals the
host result.  Invalid graphs raise and leave the context usable; no device memory is kept."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
import squidpy_b200.gr._ppatterns as pp  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from squidpy_b200._device import device_matrix, graph_args  # noqa: E402
from squidpy_b200.gr import AutocorrPlan  # noqa: E402
from tests.test_gpu_device_buffers import _settled_pool_used  # noqa: E402
from tests.test_gpu_nhood_device_graph import CuSparse  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu
KEY = "spatial_connectivities"
N_VAR = 23


def _x(n, seed=0, dtype=np.float32):
    x = sp.random(n, N_VAR, density=0.2, format="csr", random_state=seed, dtype=np.float64)
    x.data = np.round(x.data * 16) / 4
    x[:, 3] = 0.0  # an all-zero feature -> NaN scores
    x.eliminate_zeros()
    return x.astype(dtype)


def _weighted(g, seed, dtype=np.float32, signs=False):
    rng = np.random.default_rng(seed)
    v = rng.random(g.nnz) + 0.05
    if signs:
        v *= rng.choice([-1.0, 1.0], g.nnz)
    return sp.csr_matrix((v.astype(dtype), g.indices.copy(), g.indptr.copy()), shape=g.shape)


def _messy(dtype=np.float32):
    """Empty rows, explicit zeros, self-loops and negative weights in canonical rows."""
    g = synth.hex_graph(30, 40).tolil()
    g[::7] = 0
    g = (g.tocsr() + sp.eye(1200, dtype=np.float32, format="csr")).tocsr()
    g.eliminate_zeros()
    g.sort_indices()
    g = _weighted(g, 9, dtype, signs=True)
    g.data[::13] = 0.0
    return g


def _graph(kind):
    knn6 = synth.knn_graph(synth.hex_coords(30, 40) + np.random.default_rng(0).normal(0, 7, (1200, 2)), k=6)
    if kind == "hex":  # binary, <= 6 entries per row: compact rows
        return synth.hex_graph(30, 40)
    if kind == "knn_w":  # 6 different weights per row: packed rows of 8
        return _weighted(knn6, 1)
    if kind == "knn12_w":  # 12 entries: packed rows of 16
        return _weighted(synth.knn_graph(synth.hex_coords(30, 40), k=12), 2)
    if kind == "knn24_w":  # 24 entries: the CSR walk
        return _weighted(synth.knn_graph(synth.hex_coords(30, 40), k=24), 3)
    if kind == "f64":
        return _weighted(knn6, 4, np.float64)
    if kind == "long_rows":  # a few rows of 300 entries: the row sums' pairwise trees split below the top
        g = knn6.tocoo()
        rng = np.random.default_rng(6)
        long = (0, 17, 500)
        keep = ~np.isin(g.row, long)
        rows = np.concatenate([g.row[keep]] + [np.full(300, r) for r in long])
        cols = np.concatenate([g.col[keep]] + [np.sort(rng.choice(1200, 300, replace=False)) for _ in long])
        m = sp.csr_matrix((np.ones(rows.size, np.float32), (rows, cols)), shape=(1200, 1200))
        m.sort_indices()
        return _weighted(m, 7)
    if kind == "empty":
        return sp.csr_matrix((1200, 1200), dtype=np.float32)
    assert kind == "messy"
    return _messy()


# W format of each graph (0 packed 8, 1 packed 16, 2 CSR walk, 3 compact)
FORMATS = {"hex": 3, "knn_w": 0, "knn12_w": 1, "knn24_w": 2, "f64": 2, "messy": 0, "long_rows": 2, "empty": 0}


def _adata(X, w):
    var = pd.DataFrame(index=[f"g{i}" for i in range(N_VAR)])
    return AnnDataLite(X=X, obsp={KEY: w}, var=var, shape=(w.shape[0], N_VAR))


def _torch_csr(m, ip=torch.int64, ix=torch.int64):
    return torch.sparse_csr_tensor(torch.from_numpy(m.indptr.astype(np.int64)).to(ip), torch.from_numpy(m.indices.astype(np.int64)).to(ix),
                                   torch.from_numpy(m.data.copy()), size=m.shape).cuda()


def _dev(g, container):
    if container == "torch":
        return _torch_csr(g)
    ip, ix = {"cai32": (np.int32, np.int32), "cai64": (np.int64, np.int64), "cai_mixed": (np.int64, np.int32)}[container]
    return CuSparse.of(g, ip, ix)


def _snapshot(dev):
    if isinstance(dev, torch.Tensor):
        return [dev.crow_indices().clone(), dev.col_indices().clone(), dev.values().clone()]
    return [dev.indptr.t.clone(), dev.indices.t.clone(), dev.data.t.clone()]


def _frames(g_host, g_dev, x_host, x_dev=None, **kw):
    """The same X with W on the host and W on the device (X on the device when ``x_dev`` is given)."""
    x = x_host if x_dev is None else x_dev
    host = sq.gr.spatial_autocorr(_adata(x, g_host), copy=True, **kw)
    dev = sq.gr.spatial_autocorr(_adata(x, g_dev), copy=True, **kw)
    assert list(dev.index) == list(host.index)
    pd.testing.assert_frame_equal(dev, host, check_exact=True)
    return host


@pytest.fixture
def no_host_read(monkeypatch):
    """The device path must not copy the graph to the host."""

    def boom(*a, **k):
        raise AssertionError("the device graph was copied to the host")

    monkeypatch.setattr(pp, "to_host_matrix", boom)
    monkeypatch.setattr(pp, "on_host", boom)


@pytest.fixture
def host_reads(monkeypatch):
    calls = []
    real = pp.to_host_matrix

    def spy(m):
        calls.append(m)
        return real(m)

    monkeypatch.setattr(pp, "to_host_matrix", spy)
    return calls


def _branch(g_dev, transformation):
    plan = AutocorrPlan.from_device(graph_args(device_matrix(g_dev), g_dev.shape[0]), transformation)
    assert plan is not None
    try:
        return plan.w_info
    finally:
        plan.close()


@pytest.mark.parametrize("transformation", [True, False])
@pytest.mark.parametrize("kind", list(FORMATS))
def test_device_graph_equals_host_graph(kind, transformation, no_host_read):
    g = _graph(kind)
    dev = _dev(g, "cai32")
    fmt, s0_branch = _branch(dev, transformation)
    assert fmt == FORMATS[kind]
    if transformation and g.dtype == np.float32:
        assert s0_branch == 0  # a row-normalised float32 graph: S0 as an exact integer sum
    before = _snapshot(dev)
    x = _x(g.shape[0])
    for mode in ("moran", "geary"):
        _frames(g, dev, x, mode=mode, transformation=transformation)
    after = _snapshot(dev)
    assert all(torch.equal(a, b) for a, b in zip(before, after))  # the caller's graph is unchanged


def test_s0_sequential_branch(no_host_read):
    # unnormalised weights spanning 2^-60 .. 1: the parallel integer sum does not apply, one thread walks the chain
    g = _graph("knn_w").astype(np.float64)
    g.data[::5] *= 2.0**-60
    dev = _dev(g, "cai32")
    assert _branch(dev, False) == (2, 1)
    _frames(g, dev, _x(g.shape[0]), transformation=False)


@pytest.mark.parametrize("container", ["cai32", "cai64", "cai_mixed", "torch"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_index_widths_containers_and_dtypes(container, dtype, no_host_read):
    g = _graph("knn_w").astype(dtype)
    _frames(g, _dev(g, container), _x(g.shape[0]), mode="geary")


@pytest.mark.parametrize("kind", ["hex", "knn24_w"])
def test_device_x_and_permutations(kind, no_host_read):
    g = _graph(kind)
    x = _x(g.shape[0], seed=3)
    xd = torch.from_numpy(x.toarray()).cuda()
    for mode in ("moran", "geary"):
        _frames(g, _dev(g, "torch"), x, xd, mode=mode, n_perms=20, seed=7)


def _unsorted(g):
    g = g.copy()
    a, b = g.indptr[5], g.indptr[6]
    g.indices[a:b] = g.indices[a:b][::-1].copy()
    g.data[a:b] = g.data[a:b][::-1].copy()
    g.has_sorted_indices = False
    return g


def _repeated(g):
    g = g.tocoo()
    r = np.concatenate([g.row, [7]])
    c = np.concatenate([g.col, [g.col[g.row == 7][0]]])
    v = np.concatenate([g.data, [np.float32(0.5)]])
    order = np.lexsort((c, r))
    ptr = np.concatenate([[0], np.cumsum(np.bincount(r, minlength=g.shape[0]))]).astype(np.int32)
    m = sp.csr_matrix((v[order].astype(np.float32), c[order].astype(np.int32), ptr), shape=g.shape)
    m.has_canonical_format = False
    return m


def _strided(t):
    """A view of ``t`` with element stride 2 (every other entry of a buffer twice as long)."""
    buf = torch.zeros(2 * t.numel(), dtype=t.dtype, device=t.device)
    buf[::2] = t
    return buf[::2]


@pytest.mark.parametrize("case", ["csc", "int", "bool", "unsorted", "repeated", "strided_data", "strided_indices"])
def test_fallback(case, host_reads):
    g = _graph("knn_w")
    if case == "csc":
        host, dev = g.tocsc(), CuSparse.of(g.tocsc())
    elif case == "int":
        gi = sp.csr_matrix((np.arange(1, g.nnz + 1, dtype=np.int32) % 5 + 1, g.indices, g.indptr), shape=g.shape)
        host, dev = gi, CuSparse.of(gi)
    elif case == "bool":
        gb = sp.csr_matrix((np.ones(g.nnz, bool), g.indices, g.indptr), shape=g.shape)
        host = gb
        dev = CuSparse("csr", gb.indptr, gb.indices, torch.ones(g.nnz, dtype=torch.bool), gb.shape)
    elif case == "unsorted":
        host = _unsorted(g)
        dev = CuSparse.of(host)
    elif case in ("strided_data", "strided_indices"):
        host, dev = g, CuSparse.of(g)
        arr = dev.data if case == "strided_data" else dev.indices
        arr.t = _strided(arr.t)
        assert arr.__cuda_array_interface__["strides"] is not None
    else:
        host = _repeated(g)
        dev = CuSparse.of(host)
    x = _x(g.shape[0])
    ref = sq.gr.spatial_autocorr(_adata(x, host.copy()), copy=True)
    got = sq.gr.spatial_autocorr(_adata(x, dev), copy=True)
    assert len(host_reads) == 1  # the fallback copied the graph to the host once
    pd.testing.assert_frame_equal(got, ref, check_exact=True)


def test_plan_rejects_strided_values():
    g = _graph("knn_w")
    dev = CuSparse.of(g)
    dev.data.t = _strided(dev.data.t)
    with pytest.raises(ValueError, match="contiguous"):
        AutocorrPlan.from_device(graph_args(device_matrix(dev), g.shape[0]), True)


@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_weights(bad, host_reads):
    g = _graph("knn_w")
    g.data[17] = bad
    x = _x(g.shape[0])
    # sklearn's normalize rejects them: the device graph takes the host copy and raises the same error
    with pytest.raises(ValueError) as on_host:
        sq.gr.spatial_autocorr(_adata(x, g.copy()), copy=True)
    with pytest.raises(ValueError) as on_device:
        sq.gr.spatial_autocorr(_adata(x, CuSparse.of(g)), copy=True)
    assert str(on_device.value) == str(on_host.value)
    assert len(host_reads) == 1
    # not normalised, they are read on the device like any other weight
    _frames(g, CuSparse.of(g), x, transformation=False)
    assert len(host_reads) == 1


def test_invalid_graphs_raise_and_context_stays_usable():
    g = _graph("hex")
    x = _x(g.shape[0])
    bad_idx = CuSparse.of(g)
    bad_idx.indices.t[10] = g.shape[0] + 3
    with pytest.raises(ValueError, match="out of range"):
        sq.gr.spatial_autocorr(_adata(x, bad_idx), copy=True)
    bad_ptr = CuSparse.of(g)
    bad_ptr.indptr.t[100] = bad_ptr.indptr.t[99] - 1
    with pytest.raises(ValueError, match="indptr"):
        sq.gr.spatial_autocorr(_adata(x, bad_ptr), copy=True)
    _frames(g, CuSparse.of(g), x)


def test_device_mismatch_raises():
    g = _graph("hex")
    with pytest.raises(ValueError, match="weight matrix"):
        sq.gr.spatial_autocorr(_adata(_x(g.shape[0]), CuSparse.of(g)), copy=True, device=torch.cuda.device_count())


@pytest.mark.parametrize("builder", ["grid", "knn"])
def test_full_device_pipeline_equals_host_pipeline(builder, no_host_read):
    co = synth.hex_coords(40, 50) + np.random.default_rng(5).normal(0, 3, (2000, 2))
    x = _x(2000, seed=11)
    fn = sq.gr.spatial_neighbors_grid if builder == "grid" else sq.gr.spatial_neighbors_knn
    res = {}
    for where in ("host", "device"):
        ad = synth.make_adata(co if where == "host" else torch.tensor(co, device="cuda"), None, None,
                              X=x if where == "host" else _torch_csr(x))
        fn(ad, n_neighs=6)
        if where == "device":
            assert ad.obsp[KEY].layout == torch.sparse_csr and ad.obsp[KEY].is_cuda
        res[where] = sq.gr.spatial_autocorr(ad, copy=True, n_perms=10, seed=1)
    pd.testing.assert_frame_equal(res["device"], res["host"], check_exact=True)


def test_no_device_memory_kept():
    g = _graph("knn12_w")
    x = _x(g.shape[0])
    bad = CuSparse.of(g)
    bad.indices.t[4] = -1
    good = CuSparse.of(g)
    sq.gr.spatial_autocorr(_adata(x, good), copy=True)  # warm-up: first-call allocations of the context
    base = _settled_pool_used()
    for _ in range(5):
        sq.gr.spatial_autocorr(_adata(x, good), copy=True, n_perms=3, seed=0)
        with pytest.raises(ValueError):
            sq.gr.spatial_autocorr(_adata(x, bad), copy=True)
    assert _settled_pool_used() == base
