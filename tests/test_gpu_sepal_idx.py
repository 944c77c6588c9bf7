"""sepal's saturation tables built on the GPU (``sqb_sepal_idxs`` through ``_sepal.sepal_idxs``) equal ``_compute_idxs`` on the
host copies, array for array: on the golden cases, on lattices with removed spots (orphans present), and on graphs with explicit
zeros, duplicates, unsorted rows, CSC storage, int64 indices and every value dtype, from the host and from GPU memory (torch
``sparse_csr`` / ``sparse_csc`` and cupyx-style graphs), with float64, float32 and strided device coordinates.  The orphans'
argmin follows numpy's rules (first of equal distances, first NaN) in the C entry point itself; non-finite coordinates that
scikit-learn would refuse raise its error through ``sepal``, as on the host.  The ``sepal`` frames from a device graph equal
those from its host copy bit for bit; the producer streams are honoured and the context stays usable after a rejected input."""

from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
from scipy.spatial.distance import cdist

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from squidpy_b200._lib import check, default_context, load  # noqa: E402
from squidpy_b200.gr._sepal import _compute_idxs, sepal_idxs  # noqa: E402
from tests.golden.make_golden_sepal import make_case  # noqa: E402
from tests.test_gpu_autocorr_device_input import CuArray, CuSparse  # noqa: E402
from tools.sepal_idx_time import lattice  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "sepal.npz"), allow_pickle=False))


def _expected(g, co, k):
    """The host path: a CSR copy (scipy's tocsr for anything else), eliminate_zeros, _compute_idxs on float64 coordinates."""
    h = g.copy() if (sp.issparse(g) and g.format == "csr") else sp.csr_matrix(g)
    h.eliminate_zeros()
    return _compute_idxs(h, np.asarray(co, dtype=np.float64), k)


def _same(got, want):
    for a, b in zip(got, want, strict=True):
        assert a.dtype == np.int32 and a.shape == b.shape and np.array_equal(a, b)


def _torch_sparse(g):
    if g.format == "csc":
        return torch.sparse_csc_tensor(torch.as_tensor(g.indptr), torch.as_tensor(g.indices), torch.as_tensor(g.data), size=g.shape).cuda()
    return torch.sparse_csr_tensor(torch.as_tensor(g.indptr), torch.as_tensor(g.indices), torch.as_tensor(g.data), size=g.shape).cuda()


def _all_forms(g, co, k, ip=np.int32, ix=np.int32):
    """Tables of the host graph and of its device copies (torch and cupyx-style), with host and device coordinates."""
    want = _expected(g, co, k)
    _same(sepal_idxs(g, co, k), want)
    _same(sepal_idxs(CuSparse.of(g, ip, ix), torch.as_tensor(co).cuda(), k), want)
    if g.dtype != np.bool_:  # torch has no sparse bool CSR constructor path worth relying on
        _same(sepal_idxs(_torch_sparse(g), co, k), want)
    return want


def _orphans(g, k):
    h = sp.csr_matrix(g, copy=True)  # eliminate_zeros compacts the arrays in place
    h.eliminate_zeros()
    deg = np.diff(h.indptr)
    sat = deg == k
    return [i for i in np.flatnonzero(~sat) if not sat[h.indices[h.indptr[i]:h.indptr[i + 1]]].any()]


@pytest.mark.parametrize("name", ["hex", "square"])
def test_golden_cases(name):
    g, co, k, _ = make_case(name)
    want = [GOLD[f"{name}_{key}"] for key in ("sat", "sat_idx", "unsat", "unsat_idx")]
    got = _all_forms(g, co, k)
    for a, b in zip(got, want, strict=True):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("kind,side,drop", [("square", 120, 0.03), ("hex", 100, 0.05), ("square", 64, 0.3), ("hex", 40, 0.5)])
def test_lattices_with_removed_spots(kind, side, drop):
    g, co, k = lattice(kind, side, drop, seed=side)
    assert _orphans(g, k), "the case needs orphans"
    _all_forms(g, co, k)
    _all_forms(g, co, k, np.int64, np.int64)


def _tie_case():
    """A square lattice with isolated nodes (orphans) at cell centres and on edge midpoints: equidistant, in L1, from two or
    four saturated nodes, and from farther rings."""
    g, co, k = lattice("square", 12, 0.0)
    extra = np.array([[3.5, 3.5], [5.0, 6.5], [6.5, 5.0], [2.5, 7.0], [4.5, 4.5], [8.0, 8.0], [-3.0, 5.0]])
    n = g.shape[0] + len(extra)
    h = sp.csr_matrix((g.data, g.indices, np.r_[g.indptr, np.full(len(extra), g.indptr[-1])]), shape=(n, n))
    return h, np.r_[co, extra], k


def test_equidistant_orphans():
    g, co, k = _tie_case()
    want = _all_forms(g, co, k)
    sat, unsat, unsat_idx = want[0], want[2], want[3]
    d = cdist(co[unsat[-7:]], co[sat], "cityblock")
    assert (np.sort(d, axis=1)[:, 1] == d.min(1)).sum() >= 5  # ties decide most of them
    assert np.array_equal(unsat_idx[-7:], sat[d.argmin(1)])


def _abi(g, xy, k):
    """The C entry point on a host CSR and host float64 coordinates: (tables, max degree, nonfinite)."""
    ip, ix = np.ascontiguousarray(g.indptr, np.int64), np.ascontiguousarray(g.indices, np.int64)
    data = np.ascontiguousarray(g.data, np.float64)
    xy = np.ascontiguousarray(xy, np.float64)
    n = g.shape[0]
    out = [np.empty(m, np.int32) for m in (n, n * k, n, n)]
    max_deg, ns, nu, bad = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int()
    ctx = default_context()
    with ctx.lock:
        check(load().sqb_sepal_idxs(ctx.handle, n, ix.size, ip.ctypes.data, 64, ix.ctypes.data, 64, data.ctypes.data, 1, 0, 0, 0, xy.ctypes.data, 1,
                                    2, 1, 0, 0, k, C.byref(max_deg), *(o.ctypes.data for o in out), C.byref(ns), C.byref(nu), C.byref(bad)))
    s, u = ns.value, nu.value
    return (out[0][:s], out[1][: s * k].reshape(s, k), out[2][:u], out[3][:u]), max_deg.value, bad.value


def test_argmin_rules_with_nan_and_inf_coordinates():
    """numpy's argmin of the cityblock rows: the first NaN distance wins, inf - inf is NaN, ties go to the lowest position."""
    g, co, k = _tie_case()
    (sat, sat_idx, unsat, unsat_idx), most, bad = _abi(g, co, k)
    assert most == k and bad == 0
    _same((sat, sat_idx, unsat, unsat_idx), _expected(g, co, k))
    orph = np.isin(unsat, _orphans(g, k))
    assert orph.sum() == 11  # the seven isolated nodes and the lattice's four corners
    for rows, vals in (([40, 77], [np.nan, np.inf]), ([145], [np.inf]), ([30, 146], [np.inf, -np.inf]), ([147, 90], [np.nan, 0.0]),
                       ([20, 21, 150], [np.inf, -np.inf, np.inf]), ([0], [np.nan])):
        xy = co.copy()
        for r, v in zip(rows, vals):
            xy[r, r % 2] = v
        tables, most, bad = _abi(g, xy, k)
        assert most == k and bad == 1
        want = unsat_idx.copy()
        want[orph] = sat[np.argmin(cdist(xy[unsat[orph]], xy[sat], "cityblock"), axis=1)]
        _same(tables, (sat, sat_idx, unsat, want))
        with pytest.raises(ValueError) as host:
            _expected(g, xy, k)
        with pytest.raises(ValueError) as dev:
            sepal_idxs(CuSparse.of(g), torch.as_tensor(xy).cuda(), k)
        assert str(dev.value) == str(host.value)


def test_nonfinite_coordinates_that_are_never_read():
    side = 30  # a torus: every node saturated, so no coordinate is read
    idx = np.arange(side * side).reshape(side, side)
    nb = np.stack([np.roll(idx, s, axis=a) for a, s in ((1, 1), (1, -1), (0, 1), (0, -1))], -1).reshape(-1, 4)
    g = sp.csr_matrix((np.ones(nb.size), np.sort(nb, 1).ravel(), 4 * np.arange(side * side + 1)), shape=(side * side,) * 2)
    xy = np.stack(np.meshgrid(np.arange(side, dtype=float), np.arange(side, dtype=float)), -1).reshape(-1, 2)
    xy[31, 0], xy[62, 1] = np.nan, np.inf
    assert _all_forms(g, xy, 4)[2].size == 0
    g2, co2, k2 = _tie_case()
    xy2 = co2.copy()
    xy2[1, 0] = np.nan  # an unsaturated border node with a saturated neighbour: not an orphan, never compared
    _all_forms(g2, xy2, k2)


def _messy(seed=0):
    """A lattice with removed spots, then explicit zeros (0, -0.0), NaN values, duplicates, extra edges and shuffled rows (rows
    with more than k non-zero entries are cut back by _trim)."""
    g, co, k = lattice("hex", 40, 0.08, seed=seed)
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(g.shape[0]), np.diff(g.indptr))
    cols = g.indices.astype(np.int64)
    vals = np.ones(cols.size)
    vals[rng.random(cols.size) < 0.04] = np.nan
    z = rng.choice(g.shape[0], 60, replace=False)  # explicit zeros and duplicates on some rows
    rows = np.r_[rows, z, z[:20], z[20:40]]
    cols = np.r_[cols, rng.integers(0, g.shape[0], 60), (z[:20] + 1) % g.shape[0], (z[20:40] + 7) % g.shape[0]]
    vals = np.r_[vals, np.where(np.arange(60) % 2, 0.0, -0.0), np.ones(20), np.ones(20)]
    order = np.lexsort((rng.random(rows.size), rows))  # rows in order, entries shuffled within them
    rows, cols, vals = rows[order], cols[order], vals[order]
    indptr = np.r_[0, np.cumsum(np.bincount(rows, minlength=g.shape[0]))]
    return sp.csr_matrix((vals, cols.astype(np.int32), indptr.astype(np.int32)), shape=g.shape), co, k


def _trim(m, k):
    """Drop the last non-zero entries of the rows with more than k of them, keeping zeros and order."""
    keep = np.ones(m.nnz, bool)
    for i in range(m.shape[0]):
        lo, hi = m.indptr[i], m.indptr[i + 1]
        nz = np.flatnonzero(m.data[lo:hi] != 0)
        keep[lo + nz[k:]] = False
    rows = np.repeat(np.arange(m.shape[0]), np.diff(m.indptr))[keep]
    indptr = np.r_[0, np.cumsum(np.bincount(rows, minlength=m.shape[0]))]
    return sp.csr_matrix((m.data[keep], m.indices[keep], indptr), shape=m.shape)


@pytest.mark.parametrize("dtype", [np.float64, np.float32, np.int32, np.int64, np.bool_])
def test_zeros_duplicates_unsorted_rows_and_value_dtypes(dtype):
    m, co, k = _messy()
    m = _trim(m, k)
    if dtype != np.float64:
        data = m.data if np.dtype(dtype).kind == "f" else np.where(np.isnan(m.data), 3, m.data)  # NaN stays in float graphs
        m = sp.csr_matrix((data.astype(dtype), m.indices, m.indptr), shape=m.shape)
    assert _orphans(m, k)
    _all_forms(m, co, k)
    _all_forms(m, co, k, np.int64, np.int64)


@pytest.mark.parametrize("ix", [np.int32, np.int64])
def test_csc_graphs(ix):
    m, co, k = _messy(1)
    m = _trim(m, k)
    c = sp.csc_matrix((m.data, m.indices, m.indptr), shape=m.shape)  # the transpose's storage: a CSC of another graph
    c = sp.csc_matrix(_trim(sp.csr_matrix(c), k))  # rows with more than k entries trimmed again, in scipy's tocsr order
    want = _expected(c, co, k)
    _same(sepal_idxs(c, co, k), want)
    _same(sepal_idxs(CuSparse.of(c, ix, ix), co, k), want)
    _same(sepal_idxs(_torch_sparse(c), torch.as_tensor(co).cuda(), k), want)


def test_float32_and_strided_device_coordinates():
    g, co, k = lattice("square", 80, 0.04, seed=3)
    co = co * 0.37 + 11.0
    f32 = co.astype(np.float32)
    want = _expected(g, f32.astype(np.float64), k)
    _same(sepal_idxs(CuSparse.of(g), torch.as_tensor(f32).cuda(), k), want)
    wide = torch.zeros((co.shape[0], 5), dtype=torch.float64, device="cuda")
    wide[:, 1], wide[:, 3] = torch.as_tensor(co[:, 0]).cuda(), torch.as_tensor(co[:, 1]).cuda()
    _same(sepal_idxs(CuSparse.of(g), CuArray(wide[:, 1::2]), k), _expected(g, co, k))  # element strides 5 and 2
    fort = torch.as_tensor(np.asfortranarray(co)).cuda().t().contiguous().t()
    _same(sepal_idxs(_torch_sparse(g), fort, k), _expected(g, co, k))


def _adata(g, co, n_genes=5, seed=0):
    x = np.random.default_rng(seed).random((g.shape[0], n_genes))
    return AnnDataLite(X=x, obsp={"spatial_connectivities": g}, obsm={"spatial": co}, var=pd.DataFrame(index=[f"g{q}" for q in range(n_genes)]))


@pytest.mark.parametrize("kind", ["square", "hex"])
def test_sepal_frames_from_device_graphs_equal_host(kind):
    g, co, k = lattice(kind, 60, 0.05, seed=4)
    host = sq.gr.sepal(_adata(g, co), max_neighs=k, n_iter=3000, copy=True)
    for gd, cd in ((_torch_sparse(g), torch.as_tensor(co).cuda()), (CuSparse.of(g), co), (CuSparse.of(g, np.int64, np.int64), CuArray(torch.as_tensor(co).cuda()))):
        dev = sq.gr.sepal(_adata(gd, cd), max_neighs=k, n_iter=3000, copy=True)
        assert dev.equals(host)
        assert np.array_equal(dev["sepal_score"].to_numpy(), host["sepal_score"].to_numpy(), equal_nan=True)


def test_max_neighs_message_unchanged():
    g, co, _ = lattice("hex", 20, 0.1)
    for conn in (g, CuSparse.of(g), _torch_sparse(g)):
        with pytest.raises(ValueError, match=r"^Expected `max_neighs=4`, found node with `6` neighbors\.$"):
            sq.gr.sepal(_adata(conn, co), max_neighs=4, copy=True)
    h, co2, _ = lattice("square", 20, 0.0)
    h = h.tolil()
    h[25, 300] = 1.0  # an interior node (degree 4) with two more neighbours
    h[25, 301] = 1.0
    h = h.tocsr()
    for conn in (h, CuSparse.of(h)):
        with pytest.raises(ValueError, match=r"^Expected `max_neighs=4`, found node with `6` neighbors\.$"):
            sq.gr.sepal(_adata(conn, co2), max_neighs=4, copy=True)
    s, co3, _ = lattice("square", 20, 0.0)
    s = s.tolil()
    s[5, :] = 0.0
    s = s.tocsr()
    with pytest.raises(ValueError, match=r"^Expected `max_neighs=6`, found node with `4` neighbors\.$"):
        sq.gr.sepal(_adata(CuSparse.of(s), co3), max_neighs=6, copy=True)


def test_producer_streams_are_honoured():
    g, co, k = lattice("square", 300, 0.02, seed=5)
    want = _expected(g, co, k)
    s = torch.cuda.Stream()
    src = [torch.as_tensor(a).cuda() for a in (g.indptr, g.indices, g.data, co)]
    with torch.cuda.stream(s):
        dst = [torch.zeros_like(a) for a in src]
        torch.cuda._sleep(50_000_000)  # the copies below land long after the call has been issued
        for d, a in zip(dst, src):
            d.copy_(a)
    conn = CuSparse("csr", dst[0], dst[1], dst[2], g.shape, stream=s.cuda_stream)
    _same(sepal_idxs(conn, CuArray(dst[3], s.cuda_stream), k), want)
    torch.cuda.synchronize()


def test_rejected_input_leaves_context_usable():
    g, co, k = lattice("square", 30, 0.1)
    bad = g.copy()
    bad.indices = bad.indices.copy()
    bad.indices[7] = g.shape[0] + 3
    with pytest.raises(ValueError, match="index out of range"):
        sepal_idxs(CuSparse.of(bad), co, k)
    ip = g.indptr.copy()
    ip[5] = ip[6] + 1
    with pytest.raises(ValueError, match="indptr"):
        sepal_idxs(CuSparse("csr", ip, g.indices, g.data, g.shape), co, k)
    _all_forms(g, co, k)


def test_megaspot_lattice_completes():
    """1000^2 with 1 % removed: the host path's orphans x n_sat float64 matrix is ~1.5 GB; the device builds no such matrix."""
    g, co, k = lattice("square", 1000, 0.01)
    got = sepal_idxs(_torch_sparse(g), torch.as_tensor(co).cuda(), k)
    _same(got, _compute_idxs(g, co, k))
