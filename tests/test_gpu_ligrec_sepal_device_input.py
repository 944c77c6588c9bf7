"""ligrec and sepal on an expression matrix resident in device memory: the frames equal, exactly, the ones computed from the
same matrix on the host, for every supported format, dtype and index width; the golden ligrec cases give the golden results
through the device path; the caller's producer stream is honoured; invalid input raises and leaves the context usable.
cupy is not needed: the cupy-like duck types wrap torch CUDA tensors and fail if X is read on the host."""

from __future__ import annotations

import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from squidpy_b200.gr import ligrec_analysis_device  # noqa: E402
from squidpy_b200.gr._gather import OBS_MAJOR, Gathered, device_context  # noqa: E402
from tests.golden.make_golden_ligrec import CASES, make_case  # noqa: E402
from tests.test_gpu_autocorr_device_input import CuArray, CuSparse  # noqa: E402
from tests.test_gpu_ligrec_wide import perm_chunks, upload_chunk  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "ligrec.npz"), allow_pickle=False))
GENES = ["Cd4", "CD4", "Il2", "IL2RA", "Il2rb", "Il2rg", "Tgfb1", "Ccl5", "Ccr5", "Cxcl12", "Cxcr4", "Actb", "Gapdh", "Spp1", "Cd44"]
INTER = pd.DataFrame({"source": ["il2", "cd4", "ccl5", "CXCL12", "tgfb1", "nope", "Il2_Il2ra", "Il2ra_Il2rb_Il2rg", "Spp1", "Gapdh"],
                      "target": ["il2ra_il2rb", "Ccr5", "CCR5", "cxcr4", "Actb_Gapdh", "Cd4", "Cxcr4", "Ccl5", "CD44", "Spp1"],
                      "note": list("abcdefghij")})


def _x(n=700, dtype=np.float32, seed=0, special=False):
    rng = np.random.default_rng(seed)
    x = rng.poisson(0.8, (n, len(GENES))) * (rng.random((n, len(GENES))) < 0.6)
    x = x.astype(np.float64) * (1.0 if np.dtype(dtype).kind in "iu" else rng.random(x.shape) * 4)
    if special:
        x[rng.random(x.shape) < 0.01] = np.nan
        x[3, 2], x[40, 9], x[41, 10] = np.inf, -np.inf, np.inf
    return x.astype(dtype)


def _obs(n, seed=0):
    rng = np.random.default_rng(seed)
    return pd.DataFrame({"cl": pd.Categorical(rng.choice(["t", "b", "m", "n"], n))}, index=[f"c{i}" for i in range(n)])


def _dev(x, kind, ip=np.int32, ix=np.int32):
    if kind == "dense_c":
        return torch.as_tensor(x).cuda()
    if kind == "dense_f":
        return torch.as_tensor(np.asfortranarray(x)).cuda().t().contiguous().t()
    if kind == "strided":
        wide = np.zeros((x.shape[0], 2 * x.shape[1]), dtype=x.dtype)
        wide[:, ::2] = x
        return CuArray(torch.as_tensor(wide).cuda()[:, ::2])
    if kind == "cai":
        return CuArray(torch.as_tensor(x).cuda())
    if x.dtype == np.float16:  # scipy has no float16 matrices: the pattern from float32 (exact), the values in float16
        m = sp.csr_matrix(x.astype(np.float32)) if kind == "csr" else sp.csc_matrix(x.astype(np.float32))
        return CuSparse.of(m, ip, ix, np.float16)
    m = sp.csr_matrix(x) if kind in ("csr", "torch_csr") else sp.csc_matrix(x)
    if kind == "torch_csr":
        return torch.sparse_csr_tensor(torch.from_numpy(m.indptr.astype(np.int64)), torch.from_numpy(m.indices.astype(np.int64)),
                                       torch.from_numpy(m.data), size=m.shape).cuda()
    if kind == "torch_csc":
        return torch.sparse_csc_tensor(torch.from_numpy(m.indptr.astype(np.int64)), torch.from_numpy(m.indices.astype(np.int64)),
                                       torch.from_numpy(m.data), size=m.shape).cuda()
    return CuSparse.of(m, ip, ix)


def _host_for(x, kind):
    """The host twin of the device matrix: scipy for sparse kinds (explicit NaN / inf entries stay stored), numpy otherwise
    and for float16, which scipy cannot hold (toarray() of the sparse twin would be this same array)."""
    if x.dtype == np.float16:
        return x
    if kind in ("csr", "torch_csr"):
        return sp.csr_matrix(x)
    if kind in ("csc", "torch_csc"):
        return sp.csc_matrix(x)
    return x


def _ligrec_both(x, kind, ip=np.int32, ix=np.int32, raw=False, **kw):
    n = x.shape[0]
    obs, var = _obs(n), pd.DataFrame(index=GENES)
    kw = dict(interactions=INTER, n_perms=80, seed=3, copy=True, threshold=0.05) | kw

    def ad(X):
        if raw:
            return AnnDataLite(X=np.zeros((n, 2), np.float32), obs=obs, var=pd.DataFrame(index=["u", "v"]),
                               raw=AnnDataLite(X=X, obs=obs, var=var, shape=(n, len(GENES))))
        return AnnDataLite(X=X, obs=obs, var=var, shape=(n, len(GENES)))

    host = sq.gr.ligrec(ad(_host_for(x, kind)), "cl", use_raw=raw, **kw)
    dev = sq.gr.ligrec(ad(_dev(x, kind, ip, ix)), "cl", use_raw=raw, **kw)
    for key in ("means", "pvalues", "metadata"):
        a, b = host[key], dev[key]
        assert list(a.index) == list(b.index) and list(a.columns) == list(b.columns), key
        if key == "metadata":
            assert a.equals(b)
        else:
            np.testing.assert_array_equal(np.asarray(a.sparse.to_dense(), np.float64), np.asarray(b.sparse.to_dense(), np.float64))
    return host


@pytest.mark.parametrize("kind", ["csr", "csc", "torch_csr", "torch_csc", "dense_c", "dense_f", "strided", "cai"])
def test_ligrec_formats(kind):
    res = _ligrec_both(_x(), kind)
    assert np.isfinite(res["pvalues"].sparse.to_dense().to_numpy()).sum() > 10


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.float16, np.int32, np.int64])
def test_ligrec_dtypes(dtype):
    _ligrec_both(_x(dtype=dtype, seed=1), "csr")
    _ligrec_both(_x(dtype=dtype, seed=2), "dense_c")


@pytest.mark.parametrize("ip, ix", [(np.int64, np.int64), (np.int64, np.int32), (np.int32, np.int64)])
def test_ligrec_index_widths(ip, ix):
    _ligrec_both(_x(seed=4), "csr", ip, ix)
    _ligrec_both(_x(seed=5), "csc", ip, ix)


@pytest.mark.parametrize("policy", ["min", "all"])
@pytest.mark.parametrize("clusters", [None, ["t", "m"], [("n", "b"), ("b", "b")]])
def test_ligrec_raw_policies_clusters(policy, clusters):
    _ligrec_both(_x(seed=6), "csr", raw=True, complex_policy=policy, clusters=clusters, corr_method="fdr_bh")


@pytest.mark.parametrize("kind", ["csc", "torch_csc", "torch_csr", "dense_c", "dense_f", "strided"])
@pytest.mark.parametrize("clusters", [["t", "m"], [("n", "b"), ("b", "b")]])
def test_ligrec_row_subsets_every_format(kind, clusters):
    """``clusters=`` drops the cells of the other clusters: the gather takes a proper row subset in every input format."""
    _ligrec_both(_x(seed=14), kind, clusters=clusters)


def test_ligrec_gene_symbols():
    x, n = _x(seed=7), 700
    obs = _obs(n)
    var = pd.DataFrame({"sym": GENES}, index=[f"ENSG{i}" for i in range(len(GENES))])
    kw = dict(interactions=INTER, n_perms=50, seed=1, copy=True, use_raw=False, gene_symbols="sym")
    host = sq.gr.ligrec(AnnDataLite(X=x, obs=obs, var=var), "cl", **kw)
    dev = sq.gr.ligrec(AnnDataLite(X=_dev(x, "csr"), obs=obs, var=var, shape=x.shape), "cl", **kw)
    np.testing.assert_array_equal(host["pvalues"].sparse.to_dense().to_numpy(), dev["pvalues"].sparse.to_dense().to_numpy())
    np.testing.assert_array_equal(host["means"].sparse.to_dense().to_numpy(), dev["means"].sparse.to_dense().to_numpy())


@pytest.mark.parametrize("kind", ["csr", "dense_c"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_ligrec_nan_and_inf(kind, dtype):
    _ligrec_both(_x(dtype=dtype, seed=8, special=True), kind, threshold=0.0)


def test_ligrec_several_permutation_chunks():
    """48 clusters x 6000 interaction genes: the [perm][cluster][gene] means of one pass are capped at 1 GB, i.e.
    2^30 / (48 * 6000 * 8) = 466 permutations, so 500 permutations take two passes."""
    n_cls, n_genes, n_perms = 48, 6000, 500
    n = n_cls * 30
    assert len(perm_chunks(n_perms, upload_chunk(n_perms, stride=n), n_cls, n_genes)) > 1
    rng = np.random.default_rng(9)
    x = sp.random(n, n_genes, density=0.3, format="csr", random_state=rng, dtype=np.float64).astype(np.float32)
    labels = np.repeat([f"k{i:02d}" for i in range(n_cls)], 30)
    rng.shuffle(labels)
    obs = pd.DataFrame({"cl": pd.Categorical(labels)}, index=[f"c{i}" for i in range(n)])
    names = [f"G{i}" for i in range(n_genes)]
    inter = pd.DataFrame({"source": names[0::2], "target": names[1::2]})
    cats = sorted(set(labels))
    kw = dict(interactions=inter, n_perms=n_perms, seed=11, copy=True, use_raw=False, threshold=0.0,
              clusters=[(cats[i], cats[(i + 1) % n_cls]) for i in range(n_cls)])  # every cluster takes part
    var = pd.DataFrame(index=names)
    host = sq.gr.ligrec(AnnDataLite(X=x, obs=obs, var=var), "cl", **kw)
    dev = sq.gr.ligrec(AnnDataLite(X=CuSparse.of(x), obs=obs, var=var, shape=x.shape), "cl", **kw)
    np.testing.assert_array_equal(host["pvalues"].sparse.to_dense().to_numpy(), dev["pvalues"].sparse.to_dense().to_numpy())
    np.testing.assert_array_equal(host["means"].sparse.to_dense().to_numpy(), dev["means"].sparse.to_dense().to_numpy())
    assert np.isfinite(host["pvalues"].sparse.to_dense().to_numpy()).mean() > 0.5


@pytest.mark.parametrize("name", list(CASES))
def test_golden_cases_through_the_device_path(name):
    seed, n_cells, n_genes, n_cls, kind, thr, n_perms, pseed = CASES[name]
    x, cl, inter, cpairs = make_case(seed, n_cells, n_genes, n_cls, kind)
    t = torch.as_tensor(np.ascontiguousarray(x)).cuda()
    m, ctx = device_context(t, None)
    with Gathered(ctx, m, None, np.arange(n_genes), OBS_MAJOR, nan_zero=True) as g:
        res = ligrec_analysis_device(g, cl, n_cls, inter, cpairs, threshold=thr, n_perms=n_perms, seed=pseed)
    np.testing.assert_array_equal(res.pvalues, GOLD[f"{name}_pvalues"])
    np.testing.assert_array_equal(res.means, GOLD[f"{name}_means"])


# ---- sepal -------------------------------------------------------------------------------------------------------------
def _sepal_adata(X, n_var, raw=None, layers=None):
    g = synth.hex_graph(14, 15)
    var = pd.DataFrame(index=[f"g{i}" for i in range(n_var)])
    return AnnDataLite(X=X, obsp={"spatial_connectivities": g}, obsm={"spatial": synth.hex_coords(14, 15)}, var=var,
                       shape=(g.shape[0], n_var), raw=raw, layers=layers)


def _sepal_x(n, g=9, seed=0, dtype=np.float32):
    rng = np.random.default_rng(seed)
    x = (rng.random((n, g)) * 3 * (rng.random((n, g)) < 0.5)).astype(dtype)
    x[:, 3] = 0
    return x


@pytest.mark.parametrize("kind", ["csr", "csc", "torch_csr", "dense_c", "strided"])
def test_sepal_formats(kind):
    x = _sepal_x(14 * 15)
    kw = dict(max_neighs=6, n_iter=2000, copy=True, genes=["g5", "g1", "g3", "g7"])
    host = sq.gr.sepal(_sepal_adata(_host_for(x, kind), x.shape[1]), **kw)
    dev = sq.gr.sepal(_sepal_adata(_dev(x, kind), x.shape[1]), **kw)
    assert list(host.index) == list(dev.index)
    np.testing.assert_array_equal(host.to_numpy(), dev.to_numpy())


def test_sepal_integer_gene_positions():
    x = _sepal_x(14 * 15, seed=4)
    kw = dict(max_neighs=6, n_iter=2000, copy=True, genes=[5, 1, -2, 3])
    host = sq.gr.sepal(_sepal_adata(x, x.shape[1]), **kw)
    dev = sq.gr.sepal(_sepal_adata(_dev(x, "csr"), x.shape[1]), **kw)
    assert list(host.index) == list(dev.index)
    np.testing.assert_array_equal(host.to_numpy(), dev.to_numpy())
    with pytest.raises(IndexError):
        sq.gr.sepal(_sepal_adata(_dev(x, "csr"), x.shape[1]), max_neighs=6, n_iter=10, copy=True, genes=[1, 9])


def test_sepal_raw_layer_and_batches():
    n = 14 * 15
    x, xr, xl = _sepal_x(n, seed=1), _sepal_x(n, 11, seed=2, dtype=np.float64), _sepal_x(n, seed=3, dtype=np.int32)
    raw_h = AnnDataLite(X=sp.csr_matrix(xr), var=pd.DataFrame(index=[f"g{i}" for i in range(11)]))
    raw_d = AnnDataLite(X=_dev(xr, "csr"), var=pd.DataFrame(index=[f"g{i}" for i in range(11)]), shape=xr.shape)
    kw = dict(max_neighs=6, n_iter=1500, copy=True)
    host = sq.gr.sepal(_sepal_adata(x, 9, raw=raw_h), use_raw=True, **kw)
    dev = sq.gr.sepal(_sepal_adata(_dev(x, "dense_c"), 9, raw=raw_d), use_raw=True, **kw)
    assert list(host.index) == list(dev.index)
    np.testing.assert_array_equal(host.to_numpy(), dev.to_numpy())
    host = sq.gr.sepal(_sepal_adata(x, 9, layers={"L": xl}), layer="L", **kw)
    dev = sq.gr.sepal(_sepal_adata(x, 9, layers={"L": _dev(xl, "dense_c")}), layer="L", **kw)
    np.testing.assert_array_equal(host.to_numpy(), dev.to_numpy())
    # forced batches: three genes per device call
    from squidpy_b200.gr import sepal_scores
    from squidpy_b200.gr._sepal import _compute_idxs

    g = synth.hex_graph(14, 15)
    idx = _compute_idxs(g, synth.hex_coords(14, 15), 6)
    xn = x.copy()
    xn[7, 4] = np.nan  # NaN stays NaN, as on the host
    one = sepal_scores(xn, *idx, max_neighs=6, n_iter=1500)
    for b in (1, 3, 4):
        np.testing.assert_array_equal(sepal_scores(_dev(xn, "csr"), *idx, max_neighs=6, n_iter=1500, batch_genes=b), one)
        np.testing.assert_array_equal(sepal_scores(xn, *idx, max_neighs=6, n_iter=1500, batch_genes=b), one)


# ---- producer stream and errors ------------------------------------------------------------------------------------------
def test_producer_stream_is_honoured():
    x = _x(n=4000, seed=12)
    obs, var = _obs(4000), pd.DataFrame(index=GENES)
    kw = dict(interactions=INTER, n_perms=30, seed=2, copy=True, use_raw=False)
    host = sq.gr.ligrec(AnnDataLite(X=x, obs=obs, var=var), "cl", **kw)
    side = torch.cuda.Stream()
    src = torch.as_tensor(x).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)  # the copy below lands long after the call was made
        dst = torch.empty_like(src)
        dst.copy_(src)
    ev = CuArray(dst, stream=side.cuda_stream)
    dev = sq.gr.ligrec(AnnDataLite(X=ev, obs=obs, var=var, shape=x.shape), "cl", **kw)
    np.testing.assert_array_equal(host["pvalues"].sparse.to_dense().to_numpy(), dev["pvalues"].sparse.to_dense().to_numpy())


def _ligrec_dev(X, n, **kw):
    return sq.gr.ligrec(AnnDataLite(X=X, obs=_obs(n), var=pd.DataFrame(index=GENES), shape=(n, len(GENES))), "cl", interactions=INTER,
                        n_perms=10, copy=True, use_raw=False, **kw)


def test_errors_leave_the_context_usable():
    x = _x(n=300, seed=13)
    m = sp.csr_matrix(x)
    col = GENES.index("Il2")
    # duplicate entries in a gathered cell: row 0 stores Il2 (a gene of the test) twice
    x0 = x.copy()
    x0[0, col] = 2.0  # the original entry is stored too
    m0 = sp.csr_matrix(x0)
    a = m0.indptr[1]
    dup_ip = m0.indptr.astype(np.int32).copy()
    dup_ip[1:] += 1
    dup = CuSparse("csr", dup_ip, np.insert(m0.indices, a, col).astype(np.int32), np.insert(m0.data, a, np.float32(1.0)), m0.shape)
    with pytest.raises(ValueError, match="same gathered cell"):
        _ligrec_dev(dup, 300)
    # an index out of range
    bad = m.indices.astype(np.int32).copy()
    bad[m.indices == col] = len(GENES) + 5
    with pytest.raises(ValueError, match="out of range"):
        _ligrec_dev(CuSparse("csr", m.indptr.astype(np.int32), bad, m.data, m.shape), 300)
    # a decreasing indptr
    ip = m.indptr.astype(np.int64).copy()
    ip[5], ip[6] = ip[6] + 1, ip[5]
    with pytest.raises(ValueError, match="indptr"):
        _ligrec_dev(CuSparse("csr", ip, m.indices.astype(np.int32), m.data, m.shape), 300)
    # a device mismatch
    with pytest.raises(ValueError, match="does not match"):
        _ligrec_dev(_dev(x, "csr"), 300, device=torch.cuda.device_count())
    # an unsupported dtype
    with pytest.raises(TypeError, match="dtype"):
        _ligrec_dev(torch.as_tensor(x > 1).cuda(), 300)
    ms = sp.csr_matrix(_sepal_x(14 * 15))
    ips = ms.indptr.astype(np.int64).copy()
    ips[5], ips[6] = ips[6] + 1, ips[5]
    with pytest.raises(ValueError, match="indptr"):
        sq.gr.sepal(_sepal_adata(CuSparse("csr", ips, ms.indices, ms.data, ms.shape), 9), max_neighs=6, n_iter=10, copy=True)
    # the next call on the same context succeeds and equals the host result
    res = _ligrec_both(x, "csr")
    assert res["means"].shape[0] > 0
