"""Delaunay graphs on the GPU (``DelaunayBuilder``, ``spatial_neighbors_delaunay``, ``sqb_delaunay_2d``).

The expected graph is the reference builder's arithmetic restated here: ``scipy.spatial.Delaunay(coords).vertex_neighbor_vertices``,
float32 ones, ``np.linalg.norm`` distances in the coordinates' dtype, the diagonal calls, then the same post-processing.
Inputs whose triangulation is unique compare bit for bit; exactly cocircular inputs compare edge counts and symmetry (Qhull's
choice of diagonal is its own); duplicates compare once every copy is mapped to its lowest index.  Host and device paths
agree bit for bit."""

from __future__ import annotations

import json
import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
from scipy.spatial import Delaunay, QhullError

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200.gr import DelaunayBuilder, KNNBuilder, delaunay_2d  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu


def _same(a, b, what=""):
    a, b = sp.csr_matrix(a), sp.csr_matrix(b)
    a.sort_indices(), b.sort_indices()
    assert a.shape == b.shape, what
    assert a.dtype == b.dtype, (what, a.dtype, b.dtype)
    assert np.array_equal(a.indptr, b.indptr), what
    assert np.array_equal(a.indices, b.indices), what
    assert np.array_equal(a.data, b.data), what


def _to_scipy(t):
    t = t.cpu()
    return sp.csr_matrix((t.values().numpy(), t.col_indices().numpy(), t.crow_indices().numpy()), shape=tuple(t.shape))


def _uniform(n, seed=0):
    return np.random.default_rng(seed).uniform(0, 1000, (n, 2))


def _wheel(k=5000):
    t = np.arange(k) * (2 * np.pi / k)
    return np.vstack([[0.0, 0.0], np.c_[np.cos(t), np.sin(t)] * 100.0 + np.random.default_rng(3).uniform(-1e-3, 1e-3, (k, 2))])


GOLD = os.path.join(os.path.dirname(__file__), "golden", "delaunay.npz")


def _gold():
    g = np.load(GOLD)
    return g, json.loads(str(g["meta"]))


def _gm(g, key, name):
    n = g[f"{key}|{name}|indptr"].size - 1
    return sp.csr_matrix((g[f"{key}|{name}|data"], g[f"{key}|{name}|indices"], g[f"{key}|{name}|indptr"]), shape=(n, n))


_G, _META = _gold()


@pytest.mark.parametrize("c", _META["cases"], ids=[c["key"] for c in _META["cases"]])
def test_golden_cases_host_and_device(c):
    """The unmodified reference DelaunayBuilder's output, bit for bit, on both paths."""
    xy = _G[f"coords|{c['coords']}"]
    exp = _gm(_G, c["key"], "adj"), _gm(_G, c["key"], "dst")
    if c.get("library"):
        codes = _G["codes|lib"]
        ad = synth.make_adata(xy, None, None)
        ad.obs["library"] = pd.Categorical.from_codes(codes, categories=["a", "b"])
        opt = dict(c["opt"])
        got = sq.gr.spatial_neighbors_delaunay(ad, library_key="library", copy=True, **opt)
        _same(got.connectivities, exp[0]), _same(got.distances, exp[1])
        ad.obsm["spatial"] = torch.from_numpy(xy).cuda()
        got = sq.gr.spatial_neighbors_delaunay(ad, library_key="library", copy=True, **opt)
        _same(_to_scipy(got.connectivities), exp[0]), _same(_to_scipy(got.distances), exp[1])
        return
    opt = {k: (tuple(v) if isinstance(v, list) else v) for k, v in c["opt"].items()}
    got = DelaunayBuilder(**opt).build(xy)
    _same(got[0], exp[0], "adj host"), _same(got[1], exp[1], "dst host")
    if xy.dtype.kind == "f":
        dev = DelaunayBuilder(**opt).build(torch.from_numpy(xy).cuda())
        _same(_to_scipy(dev[0]), exp[0], "adj device"), _same(_to_scipy(dev[1]), exp[1], "dst device")


@pytest.mark.parametrize("e", _META["errors"], ids=[e["coords"] for e in _META["errors"]])
def test_golden_errors_both_paths(e):
    xy = _G[f"coords|{e['coords']}"]
    exc = QhullError if e["type"] == "QhullError" else ValueError
    with pytest.raises(exc) as info:
        DelaunayBuilder().build(xy)
    if exc is ValueError:
        assert str(info.value) == e["message"]
    with pytest.raises(exc):
        DelaunayBuilder().build(torch.from_numpy(xy).cuda())


def _exact_rows(name):
    return _G[f"exact|{name}|indptr"], _G[f"exact|{name}|indices"]


def _common_pairs(ip, ix):
    n = ip.size - 1
    a = sp.csr_matrix((np.ones(ix.size), ix, ip), shape=(n, n))
    return a, (a @ a).tocsr()


def _incircle_rel(p, q, r, t):
    """|exact in-circle determinant| / its permanent, in rationals."""
    from fractions import Fraction as F

    P = [(F(float(v[0])), F(float(v[1]))) for v in (p, q, r, t)]
    rows = [(a[0] - P[3][0], a[1] - P[3][1]) for a in P[:3]]
    rows = [(x, y, x * x + y * y) for x, y in rows]
    (a1, a2, a3), (b1, b2, b3), (c1, c2, c3) = rows
    det = a3 * (b1 * c2 - b2 * c1) - b3 * (a1 * c2 - a2 * c1) + c3 * (a1 * b2 - a2 * b1)
    perm = abs(a3) * (abs(b1 * c2) + abs(b2 * c1)) + abs(b3) * (abs(a1 * c2) + abs(a2 * c1)) + abs(c3) * (abs(a1 * b2) + abs(a2 * b1))
    return abs(det) / perm


def _orient_rel(p, q, r):
    from fractions import Fraction as F

    """|sin| of the angle at r between r->p and r->q: the exact orientation over the product of the two lengths."""
    (px, py), (qx, qy), (rx, ry) = [(F(float(v[0])), F(float(v[1]))) for v in (p, q, r)]
    det = (px - rx) * (qy - ry) - (py - ry) * (qx - rx)
    return float(abs(det)) / (float(np.hypot(p[0] - r[0], p[1] - r[1])) * float(np.hypot(q[0] - r[0], q[1] - r[1])))


@pytest.mark.parametrize("c", _META["cocircular"], ids=[c["coords"] for c in _META["cocircular"]])
def test_cocircular_near_cocircular_and_duplicates(c):
    """Contract items 2-5: the GPU equals the exact restatement (same perturbation, same duplicate rule) bit for bit on both
    paths, with device distances equal to the host's; against Qhull the differences are diagonals of cocircular sets (exact
    inputs), of quadrilaterals within 1e-10 of cocircular (near inputs), or the choice of a duplicate's representative."""
    name, kind = c["coords"], c["kind"]
    xy = _G[f"coords|{name}"]
    ep, ex = _exact_rows(name)
    ip, ix = delaunay_2d(xy)
    assert np.array_equal(ip, ep) and np.array_equal(ix, ex)
    host = DelaunayBuilder().build(xy)
    dev = DelaunayBuilder().build(torch.from_numpy(xy).cuda())
    _same(_to_scipy(dev[0]), host[0]), _same(_to_scipy(dev[1]), host[1])
    qp, qx = _G[f"qhull|{name}|indptr"], _G[f"qhull|{name}|indices"]
    n = xy.shape[0]
    mine, theirs = _edge_set(ip, ix), _edge_set(qp, qx)
    if kind == "dup":
        _, first, inv = np.unique(xy, axis=0, return_index=True, return_inverse=True)
        rep = first[inv.ravel()]
        assert np.all(np.diff(ip)[rep != np.arange(n)] == 0)
        assert {(rep[i], rep[j]) for i, j in mine} == {(rep[i], rep[j]) for i, j in theirs}
        return
    if kind == "exact":
        assert len(mine) == len(theirs)
    a, _ = _common_pairs(ip, ix)
    diff = [(i, j) for i, j in mine - theirs if i < j]
    print(f"{name}: {len(diff)} edges differ from Qhull")
    tol = 0 if kind == "exact" else 1e-10
    for i, j in diff:
        # a diagonal of a (nearly) cocircular quadrilateral of common neighbours, or, on near inputs, the edge of a hull sliver
        # whose third point is within round-off of the line (Qhull merges those)
        w = [k for k in a[i].indices if a[j, k]]
        ok = any(_incircle_rel(xy[i], xy[u], xy[j], xy[v]) <= tol for u in w for v in w if u < v)
        if not ok and kind == "near":
            ok = any(_orient_rel(xy[i], xy[j], xy[u]) < 1e-10 for u in w)
        assert ok, (i, j, w)


def test_reference_known_answers():
    """The reference's 4-point Delaunay graph and distances (tests/graph/test_spatial_neighbors.py) and its radius_min_max grid."""
    xy = np.array([[1, 0], [3, 0], [5, 6], [0, 4]])
    gt_ddist = np.array([[0.0, 2.0, 0.0, 4.12310563], [2.0, 0.0, 6.32455532, 5.0], [0.0, 6.32455532, 0.0, 5.38516481],
                         [4.12310563, 5.0, 5.38516481, 0.0]])
    gt_dgraph = np.array([[0.0, 1.0, 0.0, 1.0], [1.0, 0.0, 1.0, 1.0], [0.0, 1.0, 0.0, 1.0], [1.0, 1.0, 1.0, 0.0]])
    for coords in (xy, torch.from_numpy(xy.astype(np.float64)).cuda()):
        ad = synth.make_adata(xy, None, None)
        ad.obsm["spatial"] = coords
        res = sq.gr.spatial_neighbors_delaunay(ad, copy=True)
        conn, dist = (res.connectivities, res.distances) if not torch.is_tensor(coords) else (_to_scipy(res.connectivities), _to_scipy(res.distances))
        np.testing.assert_array_equal(conn.toarray(), gt_dgraph)
        np.testing.assert_allclose(dist.toarray(), gt_ddist)
        for set_diag in (False, True):
            for radius in [(0, np.inf), (2.0, 4.0), (-42, -420), (100, 200)]:
                dd, dg = gt_ddist.copy(), gt_dgraph.copy()
                minn, maxx = sorted(radius)
                mask = (dd < minn) | (dd > maxx)
                dd[mask] = 0.0
                dg[mask] = 0.0
                if set_diag:
                    dg[np.arange(4), np.arange(4)] = 1.0
                res = sq.gr.spatial_neighbors_delaunay(ad, radius=radius, set_diag=set_diag, copy=True)
                conn, dist = (res.connectivities, res.distances) if not torch.is_tensor(coords) else (_to_scipy(res.connectivities), _to_scipy(res.distances))
                np.testing.assert_array_equal(conn.toarray(), dg)
                np.testing.assert_allclose(dist.toarray(), dd)


PRED_SRC = r"""
#include "delaunay_pred.h"
__global__ void k(const double* q, int n, int* out) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const double* p = q + 8 * t;
    out[3 * t] = dpred::orient2d(p, p + 2, p + 4);
    out[3 * t + 1] = dpred::incircle(p, p + 2, p + 4, p + 6);
    out[3 * t + 2] = dpred::incircle_sos(p, p + 2, p + 4, p + 6, 3, 1, 7, 5);
}
extern "C" int run(const double* hq, int n, int* hout) {
    double* d; int* o;
    if (cudaMalloc(&d, 64 * (size_t)n) || cudaMalloc(&o, 12 * (size_t)n)) return 1;
    cudaMemcpy(d, hq, 64 * (size_t)n, cudaMemcpyHostToDevice);
    k<<<(n + 127) / 128, 128>>>(d, n, o);
    int e = (int)cudaMemcpy(hout, o, 12 * (size_t)n, cudaMemcpyDeviceToHost);
    cudaFree(d), cudaFree(o);
    return e;
}
"""


def test_device_predicates_match_rationals(tmp_path):
    """The predicates as the library builds them (sm_90a, -O3, -fmad=false) agree in sign with rational arithmetic on the
    device, on random, exactly degenerate, ulp-jittered and wide-exponent inputs."""
    import ctypes as C
    import shutil
    import subprocess

    from tests.test_delaunay_host import _inputs, incircle_q, orient_q

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    src, so = tmp_path / "p.cu", tmp_path / "p.so"
    src.write_text(PRED_SRC)
    hdr = os.path.join(os.path.dirname(__file__), "..", "squidpy_b200", "csrc")
    subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-fmad=false", "-Xcompiler", "-fPIC", "-shared",
                    "-I", hdr, str(src), "-o", str(so), "-lcudart"], check=True)
    lib = C.CDLL(str(so))
    rng = np.random.default_rng(0)
    q = np.ascontiguousarray(np.concatenate([_inputs(rng, k, 300) for k in ("random", "lattice", "ulp", "exponent")]))
    out = np.zeros((q.shape[0], 3), dtype=np.int32)
    assert lib.run(q.ctypes.data_as(C.c_void_p), C.c_int(q.shape[0]), out.ctypes.data_as(C.c_void_p)) == 0
    for (a, b, c, d), (o, ic, sos) in zip(q, out):
        assert o == orient_q(a, b, c)
        assert ic == incircle_q(a, b, c, d)
        assert sos != 0 or orient_q(a, b, c) == 0 or len({tuple(p) for p in (a, b, c, d)}) < 4


def _scipy_rows(xy):
    """scipy's vertex_neighbor_vertices with every row in ascending order."""
    rp, rx = Delaunay(xy).vertex_neighbor_vertices
    m = sp.csr_matrix((np.ones(rx.size), rx, rp), shape=(xy.shape[0],) * 2)
    m.sort_indices()
    return m.indptr, m.indices


def _edge_set(ip, ix):
    rows = np.repeat(np.arange(ip.size - 1), np.diff(ip))
    return set(zip(rows.tolist(), ix.tolist()))


def _check_qhull(xy, ip, ix):
    """Equal to Qhull, except rows where Qhull's round-off picked another diagonal of a near-cocircular quadrilateral: there
    the row equals the exact restatement on the point's 60 nearest neighbours."""
    from scipy.spatial import cKDTree

    from tests.delaunay_ref import delaunay_rows

    rp, rx = _scipy_rows(xy)
    assert ix.size == rx.size
    n = xy.shape[0]
    a = sp.csr_matrix((np.ones(ix.size), ix, ip), shape=(n, n))
    b = sp.csr_matrix((np.ones(rx.size), rx, rp), shape=(n, n))
    assert (a != a.T).nnz == 0
    rows = np.unique((a != b).nonzero()[0])
    print(f"{rows.size} rows differ from Qhull")
    assert rows.size <= 2  # 0 observed on these inputs; Qhull's round-off may flip a near-cocircular diagonal
    tree = cKDTree(xy)
    for r in rows:
        nb = np.sort(tree.query(xy[r], 60)[1])
        lp, lx = delaunay_rows(xy[nb])
        k = int(np.searchsorted(nb, r))
        assert ix[ip[r]:ip[r + 1]].tolist() == nb[lx[lp[k]:lp[k + 1]]].tolist(), r


def test_scipy_200k_uniform_and_1m_hex_lattice():
    xy = _uniform(200_000, seed=11)
    ip, ix, counts = delaunay_2d(xy, pass_counts=True)
    _check_qhull(xy, ip, ix)
    assert counts.sum() == xy.shape[0] and counts[1] > 0
    hx = synth.hex_coords(1000, 1000)
    ip, ix = delaunay_2d(hx)
    _check_qhull(hx, ip, ix)


def test_pass_two_cases():
    # disc with one far outlier, thin strip, the wheel: both passes run and the result equals scipy's
    rng = np.random.default_rng(6)
    r, t = np.sqrt(rng.uniform(0, 1, 4000)) * 100, rng.uniform(0, 2 * np.pi, 4000)
    disc = np.vstack([np.c_[r * np.cos(t), r * np.sin(t)], [[1e5, 3.0]]])
    strip = np.c_[rng.uniform(0, 1e4, 3000), rng.uniform(0, 1.0, 3000)]
    for xy in (disc, strip, _wheel()):
        ip, ix, counts = delaunay_2d(xy, pass_counts=True)
        _check_qhull(xy, ip, ix)
        assert counts[1] > 0 and counts.sum() == xy.shape[0]
    ip, _, counts = delaunay_2d(_wheel(), pass_counts=True)
    assert ip[1] - ip[0] > 1000  # the centre's star, far beyond pass 1's capacity, equals Qhull's (checked above)


def test_library_key_and_nhood_from_device_graph():
    rng = np.random.default_rng(12)
    xy = rng.uniform(0, 500, (4000, 2))
    lib = pd.Categorical.from_codes(rng.integers(0, 2, 4000), categories=["a", "b"])
    lab = synth.categorical_labels(4000, 6, seed=1)
    ad = synth.make_adata(xy, None, lab)
    ad.obs["library"] = lib
    host = sq.gr.spatial_neighbors_delaunay(ad, library_key="library", radius=40.0, copy=True)
    ad.obsm["spatial"] = torch.from_numpy(xy).cuda()
    dev = sq.gr.spatial_neighbors_delaunay(ad, library_key="library", radius=40.0, copy=True)
    _same(_to_scipy(dev.connectivities), host.connectivities)
    _same(_to_scipy(dev.distances), host.distances)
    sq.gr.spatial_neighbors_delaunay(ad)
    assert ad.uns["spatial_neighbors"]["params"] == {"coord_type": "generic", "radius": None, "transform": None}
    res = sq.gr.nhood_enrichment(ad, "cluster", n_perms=16, seed=0, copy=True)
    ad.obsp["spatial_connectivities"] = sp.csr_matrix(_to_scipy(ad.obsp["spatial_connectivities"]))
    res_h = sq.gr.nhood_enrichment(ad, "cluster", n_perms=16, seed=0, copy=True)
    assert np.array_equal(res.counts, res_h.counts)


def test_from_builder_equals_mode_functions():
    xy = _uniform(1500, seed=13)
    ad = synth.make_adata(xy, None, None)
    a = sq.gr.spatial_neighbors_from_builder(ad, DelaunayBuilder(radius=30.0), copy=True)
    b = sq.gr.spatial_neighbors_delaunay(ad, radius=30.0, copy=True)
    _same(a.connectivities, b.connectivities), _same(a.distances, b.distances)
    a = sq.gr.spatial_neighbors_from_builder(ad, KNNBuilder(n_neighs=5), copy=True)
    b = sq.gr.spatial_neighbors_knn(ad, n_neighs=5, copy=True)
    _same(a.connectivities, b.connectivities), _same(a.distances, b.distances)


