"""GPU checks of ``mask_graph``: the device predicate against the rational oracle on the degenerate case sets of
``test_mask_graph_host``; masks of kNN, radius, Delaunay and grid graphs (10^4 - 10^5 points, polygons of 10 - 10^4 vertices with
holes, MultiPolygons) against a host build of ``mask_pred.h`` that tests every boundary edge; the grid's edge cases; and device
graphs with device coordinates, bit for bit with the host path."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from squidpy_b200._adata import AnnDataLite
from tests import test_mask_graph_host as H

pytestmark = pytest.mark.gpu

pred = H.pred  # the host build of mask_pred.h (fixture)


def segment_adata(segs):
    """One observation per segment end, one connectivity per segment (2k -> 2k + 1)."""
    segs = np.asarray(segs, dtype=np.float64).reshape(-1, 4)
    m = segs.shape[0]
    n = 2 * m
    adj = sp.csr_matrix((np.ones(m, np.float32), np.arange(1, n, 2), np.r_[0, np.repeat(np.arange(1, m + 1), 2)]), shape=(n, n))
    a = AnnDataLite(shape=(n, 0))
    a.obsm["spatial"] = segs.reshape(n, 2)
    a.obsp["spatial_connectivities"] = adj
    a.obsp["spatial_distances"] = adj.copy()
    return a


def device_flags(geom, segs):
    a = segment_adata(segs)
    adj, _ = sq.gr.mask_graph(a, None, geom, copy=True)
    kept = np.zeros(a.obsp["spatial_connectivities"].nnz, dtype=bool)
    kept[adj.nonzero()[0] // 2] = True
    return kept


@pytest.mark.parametrize("name", sorted(H.LATTICE_POLYS))
def test_device_predicate_matches_oracle(name):
    geom = H.LATTICE_POLYS[name]
    rng = np.random.default_rng(11 + sorted(H.LATTICE_POLYS).index(name))
    segs = np.r_[H.edge_segments(geom), H.lattice_segments(rng, geom, 300)]
    segs = np.r_[segs, H.jitter(rng, segs)]
    np.testing.assert_array_equal(device_flags(geom, segs), H.oracle(geom, segs))


def test_device_predicate_reference_recipe_and_named_cases():
    pts = H.sdata_mask_graph_points()
    segs = np.array([np.r_[pts[i], pts[j]] for i in range(12) for j in range(12)])
    np.testing.assert_array_equal(device_flags(H.CONCAVE, segs), H.oracle(H.CONCAVE, segs))
    rng = np.random.default_rng(5)
    geom = H.star(rng)
    v = H.vertices(geom)
    segs = np.c_[rng.uniform(v.min(0) - 1, v.max(0) + 1, (400, 2)), rng.uniform(v.min(0) - 1, v.max(0) + 1, (400, 2))]
    np.testing.assert_array_equal(device_flags(geom, segs), H.oracle(geom, segs))


# ------------------------------------------------------------------------------------------------------------------------
# builder graphs against the brute-force host predicate
# ------------------------------------------------------------------------------------------------------------------------
def star_ring(rng, k, cx, cy, r):
    ang = np.sort(rng.uniform(0, 2 * np.pi, k))
    rad = r * rng.uniform(0.7, 1.0, k)
    return np.c_[cx + rad * np.cos(ang), cy + rad * np.sin(ang)]


def holed_star(rng, k, cx, cy, r, n_holes=4):
    holes = [star_ring(rng, max(k // 20, 3), cx + 0.35 * r * np.cos(a), cy + 0.35 * r * np.sin(a), 0.08 * r)
             for a in np.arange(n_holes) * 2 * np.pi / n_holes]
    return H.poly(star_ring(rng, k, cx, cy, r), *holes)


def brute_flags(pred, a, geom):
    """Within-flags of adj's entries from the host build of mask_pred.h, every boundary edge tested."""
    xy = np.asarray(a.obsm["spatial"], dtype=np.float64)
    adj = a.obsp["spatial_connectivities"]
    rows = np.repeat(np.arange(adj.shape[0]), np.diff(adj.indptr))
    return pred(geom, np.c_[xy[rows], xy[adj.indices]])


def expected(flags, a, negative):
    """The keep masks of adj's and dst's entries: the host restatement of the mask and of eliminate_zeros."""
    adj, dst = a.obsp["spatial_connectivities"], a.obsp["spatial_distances"]
    n = adj.shape[0]
    rows = np.repeat(np.arange(n), np.diff(adj.indptr))
    gone = flags if negative else ~flags
    keep_a = ~gone & (adj.data != 0)
    drows = np.repeat(np.arange(n), np.diff(dst.indptr))
    keep_d = ~np.isin(drows * n + dst.indices, rows[gone] * n + adj.indices[gone]) & (dst.data != 0)
    return keep_a, keep_d


def assert_masked(res, a, keep_a, keep_d):
    for m, src, keep in ((res[0], a.obsp["spatial_connectivities"], keep_a), (res[1], a.obsp["spatial_distances"], keep_d)):
        n = src.shape[0]
        rows = np.repeat(np.arange(n), np.diff(src.indptr))
        ip = np.r_[0, np.cumsum(np.bincount(rows[keep], minlength=n))]
        np.testing.assert_array_equal(m.indptr, ip)
        np.testing.assert_array_equal(m.indices, src.indices[keep])
        np.testing.assert_array_equal(m.data, src.data[keep])
        assert m.data.dtype == src.data.dtype and m.indices.dtype == src.indices.dtype and m.indptr.dtype == src.indptr.dtype


def graph_adata(pts, kind):
    a = AnnDataLite(shape=(len(pts), 0))
    a.obsm["spatial"] = pts
    if kind == "knn":
        sq.gr.spatial_neighbors_knn(a, n_neighs=6)
    elif kind == "radius":
        sq.gr.spatial_neighbors_radius(a, radius=1.5 * np.sqrt(1.0 / len(pts)) * 100)
    elif kind == "delaunay":
        sq.gr.spatial_neighbors_delaunay(a)
    else:
        sq.gr.spatial_neighbors_grid(a, n_neighs=6, n_rings=2, set_diag=True)
    return a


def hex_points(n):
    side = int(np.sqrt(n))
    i, j = np.meshgrid(np.arange(side), np.arange(side))
    return np.c_[(i + 0.5 * (j % 2)).ravel(), (j * np.sqrt(3) / 2).ravel()].astype(np.float64) * (100.0 / side)


CASES = [("knn", 10_000, 10), ("knn", 100_000, 300), ("radius", 10_000, 1000), ("delaunay", 50_000, 100), ("delaunay", 10_000, 10_000),
         ("grid", 10_000, 1000)]


@pytest.mark.parametrize("kind,n,k", CASES)
def test_builder_graphs_match_brute_force(pred, kind, n, k):
    rng = np.random.default_rng(n + k)
    pts = hex_points(n) if kind == "grid" else rng.uniform(0, 100, (n, 2))
    a = graph_adata(pts, kind)
    geoms = [holed_star(rng, k, 50, 50, 45), H.multi(holed_star(rng, max(k // 2, 10), 30, 50, 25), holed_star(rng, max(k // 2, 10), 75, 50, 20))]
    for geom in geoms:
        pos = sq.gr.mask_graph(a, None, geom, copy=True)
        neg = sq.gr.mask_graph(a, None, geom, negative_mask=True, copy=True)
        flags = brute_flags(pred, a, geom)
        for res, negative in ((pos, False), (neg, True)):
            assert_masked(res, a, *expected(flags, a, negative))
        adj = a.obsp["spatial_connectivities"]
        assert pos[0].nnz + neg[0].nnz == np.count_nonzero(adj.data) and pos[0].multiply(neg[0]).nnz == 0
        assert 0 < pos[0].nnz < adj.nnz


def test_grid_edge_cases(pred):
    rng = np.random.default_rng(0)
    # long boundary edges next to many short ones: a big square with a finely subdivided hole
    t = np.linspace(0, 2 * np.pi, 2000, endpoint=False)
    hole = np.c_[50 + 10 * np.cos(t), 50 + 10 * np.sin(t)]
    square = H.poly([(0, 0), (100, 0), (100, 100), (0, 100)], hole)
    tiny = H.poly([(50, 50), (50.01, 50), (50, 50.01)])  # the whole polygon inside one cell of any graph's scale
    # long graph edges spanning many cells, points outside the polygon's box, a crowded cell
    crowd = 50 + rng.normal(0, 1e-3, (3000, 2))
    pts = np.r_[rng.uniform(-50, 150, (4000, 2)), crowd, rng.uniform(49.99, 50.02, (500, 2))]
    n = len(pts)
    rows = rng.integers(0, n, 60_000)
    cols = rng.integers(0, n, 60_000)
    g = sp.csr_matrix((np.ones(60_000, np.float64), (rows, cols)), shape=(n, n))
    g.sum_duplicates()
    g.data[:] = 1.0
    a = AnnDataLite(shape=(n, 0))
    a.obsm["spatial"] = pts
    a.obsp["spatial_connectivities"] = g
    a.obsp["spatial_distances"] = g.copy()
    for geom in (square, tiny, H.HOLE_TOUCHING):
        flags = brute_flags(pred, a, geom)
        for negative in (False, True):
            assert_masked(sq.gr.mask_graph(a, None, geom, negative_mask=negative, copy=True), a, *expected(flags, a, negative))


@pytest.mark.parametrize("kind", ["knn", "delaunay", "grid"])
def test_device_graph_equals_host_path(kind):
    import torch

    rng = np.random.default_rng(1)
    pts = hex_points(20_000) if kind == "grid" else rng.uniform(0, 100, (20_000, 2))
    geom = holed_star(rng, 500, 50, 50, 45)
    b = AnnDataLite(shape=(len(pts), 0))
    b.obsm["spatial"] = torch.as_tensor(pts, device="cuda")
    {"knn": lambda: sq.gr.spatial_neighbors_knn(b, n_neighs=6), "delaunay": lambda: sq.gr.spatial_neighbors_delaunay(b),
     "grid": lambda: sq.gr.spatial_neighbors_grid(b, n_neighs=6, n_rings=2, set_diag=True)}[kind]()
    from squidpy_b200._device import to_host_matrix

    h = AnnDataLite(shape=(len(pts), 0))  # the host path on the host copy of the device graph
    h.obsm["spatial"] = pts
    for key in ("spatial_connectivities", "spatial_distances"):
        h.obsp[key] = to_host_matrix(b.obsp[key])
    for negative in (False, True):
        sq.gr.mask_graph(b, None, geom, negative_mask=negative, device=0)
        want = sq.gr.mask_graph(h, None, geom, negative_mask=negative, copy=True)
        for key, w in zip(("mask_spatial_connectivities", "mask_spatial_distances"), want):
            t = b.obsp[key]
            assert t.layout == torch.sparse_csr and t.is_cuda
            np.testing.assert_array_equal(t.crow_indices().cpu().numpy(), w.indptr)
            np.testing.assert_array_equal(t.col_indices().cpu().numpy(), w.indices)
            v = t.values().cpu().numpy()
            assert v.dtype == w.data.dtype and t.crow_indices().dtype == torch.int32
            np.testing.assert_array_equal(v.view(np.uint8), w.data.view(np.uint8))
    with pytest.raises(ValueError, match="does not match"):
        sq.gr.mask_graph(b, None, geom, device=1)


def test_device_values_dtypes_and_errors():
    import torch

    rng = np.random.default_rng(2)
    pts = rng.uniform(0, 10, (500, 2))
    a = graph_adata(pts, "knn")
    pts = pts.copy()
    pts[a.obsp["spatial_connectivities"].indices[0]] = pts[0]  # coincident neighbours: a zero-length segment
    geom = holed_star(rng, 50, 5, 5, 4.5)
    adj, dst = a.obsp["spatial_connectivities"], a.obsp["spatial_distances"].copy()
    dst.data[::7] = 0.0  # zero distances: dropped even where the edge is kept
    for dt in (np.float32, np.float64, np.int32, np.int64, np.bool_):
        c = AnnDataLite(shape=(500, 0))
        c.obsm["spatial"] = torch.as_tensor(pts, device="cuda", dtype=torch.float64)
        c.obsp["spatial_connectivities"] = torch.sparse_csr_tensor(torch.as_tensor(adj.indptr.astype(np.int64)), torch.as_tensor(adj.indices.astype(np.int64)),
                                                                   torch.as_tensor(adj.data.astype(dt)), size=(500, 500)).cuda()
        c.obsp["spatial_distances"] = torch.sparse_csr_tensor(torch.as_tensor(dst.indptr.astype(np.int64)), torch.as_tensor(dst.indices.astype(np.int64)),
                                                              torch.as_tensor(dst.data), size=(500, 500)).cuda()
        h = AnnDataLite(shape=(500, 0))
        h.obsm["spatial"] = pts
        h.obsp["spatial_connectivities"] = sp.csr_matrix((adj.data.astype(dt), adj.indices.astype(np.int64), adj.indptr.astype(np.int64)), shape=(500, 500))
        h.obsp["spatial_connectivities"].indices = adj.indices.astype(np.int64)
        h.obsp["spatial_connectivities"].indptr = adj.indptr.astype(np.int64)
        h.obsp["spatial_distances"] = dst
        got = sq.gr.mask_graph(c, None, geom, copy=True)
        want = sq.gr.mask_graph(h, None, geom, copy=True)
        assert got[0].crow_indices().dtype == torch.int64 and want[0].indptr.dtype == np.int64
        for t, w in zip(got, want):
            np.testing.assert_array_equal(t.col_indices().cpu().numpy(), w.indices)
            np.testing.assert_array_equal(t.values().cpu().numpy(), w.data)
        assert (want[1].data != 0).all()
    bad = AnnDataLite(shape=(500, 0))
    xy = torch.as_tensor(pts, device="cuda").clone()
    xy[7, 0] = float("nan")
    bad.obsm["spatial"] = xy
    bad.obsp["spatial_connectivities"], bad.obsp["spatial_distances"] = c.obsp["spatial_connectivities"], c.obsp["spatial_distances"]
    with pytest.raises(ValueError, match="observation 7 are not finite"):
        sq.gr.mask_graph(bad, None, geom)
    dup = torch.sparse_csr_tensor(torch.tensor([0, 2] + [2] * 499, dtype=torch.int32), torch.tensor([3, 3], dtype=torch.int32),
                                  torch.ones(2), size=(500, 500)).cuda()
    bad.obsm["spatial"] = c.obsm["spatial"]
    bad.obsp["spatial_connectivities"] = dup
    bad.obsp["spatial_distances"] = dup
    with pytest.raises(ValueError, match="more than once"):
        sq.gr.mask_graph(bad, None, geom)
