"""ligrec's observed statistics and the gather on a device-resident X, pinned at their dispatch edges.

* ``sqb_ligrec_observed`` (csrc/dense.cu) at every warps-per-block variant of its launch rule (``observed_warps``: 4 warps up
  to 90 clusters, the opt-in attribute from 20, 3 warps from 91, 2 from 122, 1 from 182 to 363, refused from 364) and with
  ragged gene tails: the means equal pandas' ``groupby(...).mean()`` and the Kahan restatement bit for bit, the positive
  counts and sizes exactly, on data where a plain sum, a Kahan sum without its NaN reset and a ``v >= 0`` count all differ
  (``tests/test_ligrec_observed_spec.py``).
* ``sq.gr.ligrec`` from device X equals host X at 20-227 clusters; at 228 both refuse alike.
* ``sqb_dense_gather_device`` converts exactly as ``astype(float64)`` (or keeps the dtype) on int64 beyond 2^53, int32
  extremes, float16 / float32 subnormals, maxima, +-inf, NaN and stored -0.0, for every input format and both layouts.
"""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from squidpy_b200._lib import check, load  # noqa: E402
from squidpy_b200.gr._gather import GENE_MAJOR, OBS_MAJOR, Gathered, device_context  # noqa: E402
from tests.device_attrs import H100_SMEM_OPTIN, smem_optin  # noqa: E402
from tests.test_gpu_autocorr_device_input import CuSparse  # noqa: E402
from tests.test_gpu_ligrec_sepal_device_input import _dev, _host_for  # noqa: E402
from tests.test_ligrec_device_selection import kahan_group_mean  # noqa: E402
from tests.test_ligrec_observed_spec import cluster_counts, fill, observed_case, observed_warps, pandas_group_mean  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:invalid value encountered:RuntimeWarning")]  # inf - inf

OBSERVED_CLUSTERS = (19, 20, 90, 91, 121, 122, 181, 182, 227, 300, 363)
N_CELLS = 3000


@pytest.fixture(scope="module")
def optin():
    """The device's opt-in shared memory per block; the cases are written for an H100's."""
    v = smem_optin()
    if v != H100_SMEM_OPTIN:
        pytest.skip(f"the cluster counts are the H100's launch-rule boundaries ({H100_SMEM_OPTIN} B); this device has {v} B")
    return v


def _observed_cases():
    for n_cls in OBSERVED_CLUSTERS:
        wpb = observed_warps(n_cls, H100_SMEM_OPTIN)[0]
        for n_genes in sorted({1, 31, 32 * wpb - 1, 32 * wpb + 1, 1000}):  # full and ragged last blocks
            yield pytest.param(n_cls, wpb, n_genes, id=f"C{n_cls}-wpb{wpb}-G{n_genes}")


def observed_on_device(g: Gathered, codes: np.ndarray, n_cls: int):
    """``sqb_ligrec_observed`` as ``ligrec_analysis_device`` calls it: (means, positive counts, sizes)."""
    lib = load()
    c = np.ascontiguousarray(codes, dtype=np.int32)
    mean = np.empty((n_cls, g.n_genes), dtype=np.float64)
    npos = np.empty((n_cls, g.n_genes), dtype=np.int64)
    sizes = np.empty(n_cls, dtype=np.int64)
    with g.ctx.lock:
        check(lib.sqb_ligrec_observed(g.handle, c.ctypes.data, int(n_cls), mean.ctypes.data, npos.ctypes.data, sizes.ctypes.data))
    return mean, npos, sizes


def _same_bits(got: np.ndarray, expected: np.ndarray, what: str):
    assert got.shape == expected.shape and got.dtype == expected.dtype, what
    u = {2: np.uint16, 4: np.uint32, 8: np.uint64}[got.itemsize]
    bad = np.ascontiguousarray(got).view(u) != np.ascontiguousarray(expected).view(u)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} values differ in their bits, first at {i}: "
                             f"{got[i]!r} != {expected[i]!r}")


def _check_observed(g: Gathered, x0: np.ndarray, codes: np.ndarray, n_cls: int):
    mean, npos, sizes = observed_on_device(g, codes, n_cls)
    _same_bits(mean, kahan_group_mean(x0, codes, n_cls), "means vs the Kahan restatement")
    _same_bits(mean, pandas_group_mean(x0, codes, n_cls), "means vs pandas")
    np.testing.assert_array_equal(npos, cluster_counts(x0 > 0, codes, n_cls))
    np.testing.assert_array_equal(sizes, np.bincount(codes, minlength=n_cls))


@pytest.mark.parametrize("n_cls,wpb,n_genes", list(_observed_cases()))
def test_observed_kernel_every_launch_shape(optin, n_cls, wpb, n_genes):
    assert observed_warps(n_cls, optin) is not None
    got_wpb, smem, needs_attr = observed_warps(n_cls, optin)
    assert got_wpb == wpb and needs_attr == (n_cls >= 20) and smem <= optin
    x, codes = observed_case(np.random.default_rng(n_cls * 1009 + n_genes), N_CELLS, n_genes, n_cls)
    m, ctx = device_context(torch.as_tensor(x).cuda(), None)
    with Gathered(ctx, m, None, np.arange(n_genes), OBS_MAJOR, nan_zero=True) as g:
        _check_observed(g, fill(x), codes, n_cls)


def test_observed_kernel_refuses_364_clusters_and_the_context_survives(optin):
    assert observed_warps(364, optin) is None and observed_warps(363, optin)[0] == 1
    x, codes = observed_case(np.random.default_rng(364), N_CELLS, 40, 364)
    m, ctx = device_context(torch.as_tensor(x).cuda(), None)
    with Gathered(ctx, m, None, np.arange(40), OBS_MAJOR, nan_zero=True) as g:
        with pytest.raises(NotImplementedError, match="364 clusters exceed the shared-memory accumulators"):
            observed_on_device(g, codes, 364)
        merged = np.minimum(codes, 362).astype(np.int32)  # clusters 362 and 363 as one: 363 clusters, every one present
        _check_observed(g, fill(x), merged, 363)


# ---- end to end: sq.gr.ligrec from device X == host X --------------------------------------------------------------------
def _ligrec_case(n_cls: int, dtype, seed: int, n_genes: int = 37):
    x, codes = observed_case(np.random.default_rng(seed), 30 * n_cls, n_genes, n_cls, dtype, threshold=0.5)
    labels = np.array([f"k{i:03d}" for i in range(n_cls)])[codes]
    obs = pd.DataFrame({"cl": pd.Categorical(labels)}, index=[f"c{i}" for i in range(x.shape[0])])
    names = [f"G{i}" for i in range(n_genes)]
    inter = pd.DataFrame({"source": names, "target": [names[(7 * i + 3) % n_genes] for i in range(n_genes)]})
    cats = sorted(set(labels))
    ring = [(cats[i], cats[(i + 1) % n_cls]) for i in range(n_cls)]  # every cluster stays selected
    kw = dict(interactions=inter, n_perms=100, seed=seed, copy=True, use_raw=False, threshold=0.5, clusters=ring)
    return x, obs, pd.DataFrame(index=names), kw


def _dense(frame: pd.DataFrame) -> np.ndarray:
    return np.asarray(frame.sparse.to_dense(), dtype=np.float64)


@pytest.mark.parametrize("kind,dtype", [("csr", np.float32), ("strided", np.float64)])
@pytest.mark.parametrize("n_cls,wpb", [(20, 4), (91, 3), (122, 2), (182, 1), (227, 1)])
def test_ligrec_device_x_equals_host_x(optin, n_cls, wpb, kind, dtype):
    assert observed_warps(n_cls, optin)[0] == wpb
    x, obs, var, kw = _ligrec_case(n_cls, dtype, seed=n_cls)
    host = sq.gr.ligrec(AnnDataLite(X=_host_for(x, kind), obs=obs, var=var), "cl", **kw)
    dev = sq.gr.ligrec(AnnDataLite(X=_dev(x, kind), obs=obs, var=var, shape=x.shape), "cl", **kw)
    for key in ("means", "pvalues"):
        assert list(host[key].index) == list(dev[key].index) and list(host[key].columns) == list(dev[key].columns)
        np.testing.assert_array_equal(_dense(dev[key]), _dense(host[key]), err_msg=key)
    means, pv = _dense(dev["means"]), _dense(dev["pvalues"])
    assert np.isfinite(pv).sum() >= 10  # tested pairs
    assert ((means > 0) & np.isnan(pv)).sum() >= 10  # pairs with positive means that the expression-fraction mask rejects
    assert ((pv > 0) & (pv < 1)).any()


def test_ligrec_228_clusters_fail_alike_from_device_and_host_x(optin):
    """228 clusters: the observed kernel takes them (one warp per block), the permutation counts do not; device X and host X
    raise the same error."""
    assert observed_warps(228, optin)[0] == 1 and 4 * 228 * 32 * 8 > optin
    x, obs, var, kw = _ligrec_case(228, np.float32, seed=228, n_genes=9)
    kw["n_perms"] = 10
    errors = []
    for X in (x, _dev(x, "csr")):
        with pytest.raises(NotImplementedError, match="228 clusters exceed the shared-memory accumulators") as e:
            sq.gr.ligrec(AnnDataLite(X=X, obs=obs, var=var, shape=x.shape), "cl", **kw)
        errors.append(str(e.value).split(": ", 1)[1])  # without the entry point's name
    assert errors[0] == errors[1]


# ---- the gather's conversion on edge values -----------------------------------------------------------------------------
EDGES = {
    np.int64: [2**53 + 1, 2**53 + 3, -(2**53 + 1), 2**63 - 1, -(2**63)],  # round to nearest even above 2^53
    np.int32: [np.iinfo(np.int32).min, np.iinfo(np.int32).max],
    np.float16: [np.finfo(np.float16).smallest_subnormal, 65504.0, np.inf, -np.inf, np.nan, -0.0],
    np.float32: [np.finfo(np.float32).smallest_subnormal, np.finfo(np.float32).max, np.inf, -np.inf, np.nan, -0.0],
    np.float64: [np.finfo(np.float64).smallest_subnormal, np.finfo(np.float64).max, np.inf, -np.inf, np.nan, -0.0],
}
FORMATS = ("csr", "csc", "torch_csr", "torch_csc", "dense_c", "dense_f", "strided")


def _edge_matrix(dtype, rng, shape=(37, 29)):
    """Random values of ``dtype`` (40 % zeros) with every edge value planted three times; for sparse input: which entries are
    stored (every non-zero, NaN and -0.0, and some +0.0)."""
    dtype = np.dtype(dtype)
    if dtype.kind == "i":
        info = np.iinfo(dtype)
        x = rng.integers(info.min, info.max, shape, dtype=dtype, endpoint=True)
    else:
        x = (rng.standard_normal(shape) * 10.0 ** rng.integers(-3, 4, shape)).astype(dtype)
    x[rng.random(shape) < 0.4] = 0
    flat = x.reshape(-1)
    spots = rng.permutation(flat.size)
    for i, v in enumerate(EDGES[dtype.type]):
        flat[spots[3 * i : 3 * i + 3]] = v
    stored = (x != 0) | (rng.random(shape) < 0.1)
    if dtype.kind == "f":
        stored |= np.isnan(x) | np.signbit(x)
    return x, stored


def _compressed(x, stored, csr: bool, rng, shuffle: bool):
    """indptr, indices and values of the stored entries (CSR or CSC), optionally in a random order inside each segment."""
    a, s = (x, stored) if csr else (x.T, stored.T)
    major, minor = np.nonzero(s)
    indptr = np.concatenate([[0], np.cumsum(s.sum(1))])
    if shuffle:
        order = np.concatenate([indptr[i] + rng.permutation(indptr[i + 1] - indptr[i]) for i in range(a.shape[0])]).astype(np.int64)
        major, minor = major[order], minor[order]
    return indptr, minor, a[major, minor]


def _device_edge_matrix(x, stored, kind, rng):
    if kind.startswith("dense") or kind == "strided":
        return _dev(x, kind)
    csr = kind.endswith("csr")
    if kind in ("csr", "csc"):  # int32 CSR with unsorted segments, int64-indptr CSC
        ip, ix, v = _compressed(x, stored, csr, rng, shuffle=True)
        return CuSparse(kind, ip.astype(np.int32 if csr else np.int64), ix.astype(np.int32), v, x.shape)
    ip, ix, v = _compressed(x, stored, csr, rng, shuffle=False)
    make = torch.sparse_csr_tensor if csr else torch.sparse_csc_tensor
    return make(torch.from_numpy(ip.astype(np.int64)), torch.from_numpy(ix.astype(np.int64)), torch.from_numpy(v), size=x.shape).cuda()


def _expected(x, rows, cols, layout, nan_zero, keep):
    e = (x if rows is None else x[rows])[:, cols].astype(x.dtype if keep else np.float64)
    if nan_zero and e.dtype.kind == "f":
        e[np.isnan(e)] = 0.0
    return e if layout == OBS_MAJOR else e.T


def _same_values(got, expected, what):
    """Every non-NaN value bit for bit (the sign of -0.0 counts); NaN positions only (the payload is not kept)."""
    if expected.dtype.kind != "f":
        assert got.dtype == expected.dtype, what
        np.testing.assert_array_equal(got, expected, err_msg=what)
        return
    nan = np.isnan(expected)
    np.testing.assert_array_equal(np.isnan(got), nan, err_msg=what)
    _same_bits(np.where(nan, 0, got).astype(got.dtype), np.where(nan, 0, expected).astype(expected.dtype), what)


@pytest.mark.parametrize("dtype", list(EDGES), ids=lambda d: np.dtype(d).name)
@pytest.mark.parametrize("kind", FORMATS)
def test_gather_converts_edge_values_exactly(kind, dtype):
    rng = np.random.default_rng(FORMATS.index(kind) * 10 + list(EDGES).index(dtype))
    x, stored = _edge_matrix(dtype, rng)
    if np.dtype(dtype).kind == "f" and not kind.startswith("dense") and kind != "strided":
        assert (stored & (x == 0) & np.signbit(x)).any() and (stored & (x == 0) & ~np.signbit(x)).any()  # stored -0.0 and +0.0
    m, ctx = device_context(_device_edge_matrix(x, stored, kind, rng), None)
    selections = [(None, np.arange(x.shape[1])),
                  (np.sort(rng.choice(x.shape[0], 23, replace=False)), rng.permutation(x.shape[1])[:20])]  # unsorted columns
    for rows, cols in selections:
        for layout in (OBS_MAJOR, GENE_MAJOR):
            for nan_zero in (False, True):
                for keep in (False, True):
                    with Gathered(ctx, m, rows, cols, layout, nan_zero=nan_zero, keep_dtype=keep) as g:
                        got = g.download()
                    what = f"rows={'subset' if rows is not None else 'all'} layout={layout} nan_zero={nan_zero} keep_dtype={keep}"
                    _same_values(got, _expected(x, rows, cols, layout, nan_zero, keep), what)
