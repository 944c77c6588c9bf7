"""CPU checks of ``mask_graph``: the predicate of ``csrc/mask_pred.h`` (built for the host with g++, every boundary edge tested)
agrees with the rational oracle ``tests/mask_ref.py`` on random, lattice-aligned, vertex-grazing, boundary-hugging, touching and
ulp-jittered segments; and the host logic (keys, ``uns``, ``copy``, zero elimination, refusals) with the device call replaced by
a restatement built on the oracle."""

from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from squidpy_b200._adata import AnnDataLite
from squidpy_b200.gr import _mask
from tests import mask_ref

HDR = os.path.join(os.path.dirname(__file__), "..", "squidpy_b200", "csrc", "mask_pred.h")
SRC = r"""
#include "mask_pred.h"
#include <vector>
// flags[k] = segment k (seg[4k .. 4k + 3] = px, py, qx, qy) within the polygon, every boundary edge tested
extern "C" void t_within(const double* xy, const long long* ptr, const unsigned char* hole, long long n_rings, const double* seg, long long m,
                         int* flags) {
    std::vector<mpred::Edge> E;
    for (long long r = 0; r < n_rings; ++r) {
        const long long b = ptr[r], k = ptr[r + 1] - b;
        std::vector<double> scratch(2 * k + 2);
        std::vector<mpred::Edge> out(k + 1);
        out.resize(mpred::ring_edges(xy + 2 * b, k, hole[r] != 0, scratch.data(), out.data()));
        E.insert(E.end(), out.begin(), out.end());
    }
    const long long ne = (long long)E.size();
    const auto edge = [&](int64_t k) { return E[k]; };
    const auto scan = [&](auto f) { f(ne, edge); };
    const auto near = [&](double, double, auto f) { f(ne, edge); };
    for (long long s = 0; s < m; ++s) {
        const double* g = seg + 4 * s;
        const int cp = mpred::classify_point(g[0], g[1], ne, edge), cq = mpred::classify_point(g[2], g[3], ne, edge);
        flags[s] = mpred::segment_within(g[0], g[1], cp, g[2], g[3], cq, scan, near);
    }
}
"""


class Geo:
    """A minimal ``__geo_interface__`` geometry (what shapely's Polygon / MultiPolygon expose)."""

    def __init__(self, kind, coordinates):
        self.__geo_interface__ = {"type": kind, "coordinates": coordinates}


def poly(shell, *holes):
    return Geo("Polygon", (tuple(map(tuple, shell)), *(tuple(map(tuple, h)) for h in holes)))


def multi(*polys):
    return Geo("MultiPolygon", tuple(p.__geo_interface__["coordinates"] for p in polys))


@pytest.fixture(scope="module")
def pred():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    d = tempfile.mkdtemp()
    src, so = os.path.join(d, "m.cpp"), os.path.join(d, "m.so")
    with open(src, "w") as f:
        f.write(SRC)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.dirname(HDR), src, "-o", so], check=True)
    lib = C.CDLL(so)
    lib.t_within.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p]

    def within(geom, segs):
        xy, ptr, hole = _mask.polygon_rings(geom)
        s = np.ascontiguousarray(segs, dtype=np.float64).reshape(-1, 4)
        out = np.zeros(s.shape[0], dtype=np.int32)
        lib.t_within(xy.ctypes.data, ptr.ctypes.data, hole.ctypes.data, hole.size, s.ctypes.data, s.shape[0], out.ctypes.data)
        return out.astype(bool)

    yield within
    shutil.rmtree(d, ignore_errors=True)


def oracle(geom, segs):
    edges = mask_ref.boundary_edges(mask_ref.polygon_rings(geom))
    return np.array([mask_ref.segment_within(s[:2], s[2:], edges) for s in np.asarray(segs, dtype=np.float64).reshape(-1, 4)], dtype=bool)


# ------------------------------------------------------------------------------------------------------------------------
# polygons (all valid) and segments
# ------------------------------------------------------------------------------------------------------------------------
CONCAVE = poly([(0, 0), (4, 0), (4, 8), (2, 1.5), (0, 8)])  # the reference's sdata_mask_graph polygon
COMB = poly([(0, 0), (6, 0), (6, 6), (4, 6), (4, 2), (2, 2), (2, 6), (0, 6), (0, 0)])
SQUARE_HOLE = poly([(0, 0), (8, 0), (8, 8), (0, 8)], [(3, 3), (3, 5), (5, 5), (5, 3)])
HOLE_TOUCHING = poly([(0, 0), (8, 0), (8, 8), (0, 8)], [(4, 0), (5, 2), (3, 2)])  # the hole touches the shell at (4, 0)
PARTS_TOUCHING = multi(poly([(0, 0), (2, 0), (2, 2), (0, 2)]), poly([(2, 2), (4, 2), (4, 4), (2, 4)]))  # parts meet at (2, 2)
REPEATED = poly([(0, 0), (0, 0), (6, 0), (6, 0), (6, 6), (4, 6), (4, 2), (4, 2), (2, 2), (2, 6), (0, 6), (0, 0), (0, 0)])
CW_SHELL = poly([(0, 0), (0, 8), (8, 8), (8, 0)], [(3, 3), (5, 3), (5, 5), (3, 5)])  # clockwise shell, counter-clockwise hole
EMPTY = Geo("Polygon", ())


def star(rng, k=24, hole=True):
    ang = np.sort(rng.uniform(0, 2 * np.pi, k))
    rad = rng.uniform(3, 6, k)
    shell = np.c_[rad * np.cos(ang), rad * np.sin(ang)] + 6
    holes = [np.array([(5.5, 5.5), (6.5, 5.6), (6.0, 6.7)])] if hole else []
    return poly(shell, *holes)


LATTICE_POLYS = {"concave": CONCAVE, "comb": COMB, "square_hole": SQUARE_HOLE, "hole_touching": HOLE_TOUCHING, "parts_touching": PARTS_TOUCHING,
                 "repeated": REPEATED, "cw_shell": CW_SHELL}


def vertices(geom):
    return np.concatenate([np.asarray(r) for r in mask_ref.polygon_rings(geom)])


def lattice_segments(rng, geom, m, step=0.5):
    v = vertices(geom)
    lo, hi = v.min(0) - 1, v.max(0) + 1
    grid = lambda k: np.round(rng.uniform(lo, hi, (k, 2)) / step) * step  # noqa: E731
    p = grid(m)
    q = grid(m)
    # a third of the end points are polygon vertices: segments through and along the boundary, from vertex to vertex
    sel = rng.random(m) < 0.33
    p[sel] = v[rng.integers(0, len(v), sel.sum())]
    sel = rng.random(m) < 0.33
    q[sel] = v[rng.integers(0, len(v), sel.sum())]
    return np.c_[p, q]


def edge_segments(geom):
    """Every pair of vertices (along edges, across the polygon, through touching points), midpoints of edges, and zero-length
    segments at vertices and edge midpoints."""
    v = np.unique(vertices(geom), axis=0)
    pairs = [(a, b) for a in v for b in v]
    mids = []
    for ring in mask_ref.polygon_rings(geom):
        r = np.asarray(ring)
        mids += list((r + np.roll(r, -1, axis=0)) / 2)
    mids = np.asarray(mids)
    pairs += [(a, b) for a in mids for b in v] + [(a, a) for a in mids]
    return np.array([np.r_[a, b] for a, b in pairs])


def jitter(rng, segs, ulps=2):
    """Coordinates moved by up to ``ulps`` units in the last place; zeros stay (their neighbours are subnormal, outside the
    exact range)."""
    steps = rng.integers(-ulps, ulps + 1, segs.shape) * (segs != 0)
    out = segs.copy()
    for s in range(1, ulps + 1):
        out = np.where(steps >= s, np.nextafter(out, np.inf), np.where(steps <= -s, np.nextafter(out, -np.inf), out))
    return out


@pytest.mark.parametrize("name", sorted(LATTICE_POLYS))
def test_lattice_and_vertex_segments(pred, name):
    geom = LATTICE_POLYS[name]
    rng = np.random.default_rng(sorted(LATTICE_POLYS).index(name))
    segs = np.r_[edge_segments(geom), lattice_segments(rng, geom, 300)]
    want = oracle(geom, segs)
    np.testing.assert_array_equal(pred(geom, segs), want)
    assert 0 < want.sum() < want.size


@pytest.mark.parametrize("name", sorted(LATTICE_POLYS))
def test_ulp_jittered_segments(pred, name):
    geom = LATTICE_POLYS[name]
    rng = np.random.default_rng(7 + sorted(LATTICE_POLYS).index(name))
    segs = jitter(rng, np.r_[edge_segments(geom)[::3], lattice_segments(rng, geom, 150)])
    np.testing.assert_array_equal(pred(geom, segs), oracle(geom, segs))


def test_ulp_jittered_polygon(pred):
    rng = np.random.default_rng(3)
    for base in (COMB, CONCAVE, SQUARE_HOLE):
        rings = mask_ref.polygon_rings(base)
        moved = [[tuple(jitter(rng, np.asarray(p, dtype=np.float64))) for p in ring] for ring in rings]
        geom = poly(moved[0], *moved[1:])
        segs = np.r_[edge_segments(base)[::2], lattice_segments(rng, base, 100)]
        np.testing.assert_array_equal(pred(geom, segs), oracle(geom, segs))


@pytest.mark.parametrize("seed", range(4))
def test_random_segments_star_polygons(pred, seed):
    rng = np.random.default_rng(seed)
    geom = star(rng)
    v = vertices(geom)
    lo, hi = v.min(0) - 1, v.max(0) + 1
    short = rng.uniform(lo, hi, (200, 2))
    segs = np.r_[np.c_[rng.uniform(lo, hi, (200, 2)), rng.uniform(lo, hi, (200, 2))], np.c_[short, short + rng.normal(0, 0.7, (200, 2))],
                 np.c_[v[rng.integers(0, len(v), 100)], rng.uniform(lo, hi, (100, 2))]]
    want = oracle(geom, segs)
    np.testing.assert_array_equal(pred(geom, segs), want)
    assert 0 < want.sum() < want.size


def test_named_degeneracies(pred):
    cases = [
        (SQUARE_HOLE, (0, 0, 8, 0), False),  # entirely along the boundary
        (SQUARE_HOLE, (0, 0, 8, 8), False),  # through the hole
        (SQUARE_HOLE, (0, 0, 3, 3), True),  # boundary to boundary through the interior
        (SQUARE_HOLE, (1, 1, 1, 1), True),  # zero length, interior
        (SQUARE_HOLE, (0, 4, 0, 4), False),  # zero length, on the boundary
        (SQUARE_HOLE, (1, 3, 7, 3), True),  # along a hole edge (boundary) with interior on both sides
        (SQUARE_HOLE, (1, 2, 7, 2), True),  # parallel to the hole, inside
        (COMB, (1, 2, 5, 2), True),  # grazes the reflex corners (2, 2) and (4, 2) from inside
        (COMB, (1, 3, 5, 3), False),  # crosses the notch
        (COMB, (2, 2, 4, 2), False),  # the notch's bottom edge
        (CONCAVE, (1, 4, 3, 4), False),  # across the notch of the reference's polygon
        (HOLE_TOUCHING, (3, 0, 5, 0), False),  # along the shell through the touching point
        (HOLE_TOUCHING, (4, 0, 4, 3), False),  # from the touching point through the hole
        (HOLE_TOUCHING, (4, 0, 2, 1), True),  # from the touching point into the interior
        (PARTS_TOUCHING, (1, 1, 3, 3), True),  # from one part into the other through the touching point
        (PARTS_TOUCHING, (1, 3, 3, 1), False),  # through the touching point across the gaps
        (EMPTY, (0, 0, 1, 1), False),
        (EMPTY, (0, 0, 0, 0), False),
    ]
    got = np.concatenate([pred(g, [s]) for g, s, _ in cases])
    np.testing.assert_array_equal(got, [w for _, _, w in cases])
    np.testing.assert_array_equal(oracle(SQUARE_HOLE, [s for g, s, _ in cases[:7]]), [w for _, _, w in cases[:7]])


def sdata_mask_graph_points():
    """The reference's ``sdata_mask_graph`` recipe (tests/conftest.py): 12 points in four clusters, drawn by default_rng(42)."""
    rng = np.random.default_rng(42)
    return np.concatenate([rng.uniform((3.2, 4.2), (3.8, 5.2), (3, 2)), rng.uniform((0.2, 4.2), (0.8, 5.2), (3, 2)),
                           rng.uniform((1, 0.5), (3, 1.5), (3, 2)), rng.uniform((1, 5), (2, 6), (3, 2))], axis=0)


def test_reference_recipe_all_pairs(pred):
    pts = sdata_mask_graph_points()
    segs = np.array([np.r_[pts[i], pts[j]] for i in range(len(pts)) for j in range(len(pts))])
    want = oracle(CONCAVE, segs)
    np.testing.assert_array_equal(pred(CONCAVE, segs), want)
    assert 0 < want.sum() < want.size


# ------------------------------------------------------------------------------------------------------------------------
# host logic, the device call replaced by the oracle
# ------------------------------------------------------------------------------------------------------------------------
def restated(adj, dst, xy, rings, negative, *, device=None):
    """``host_mask`` restated: oracle flags per adj entry, the same positions dropped from dst, then scipy's eliminate_zeros."""
    xyr, ptr, hole = rings
    ring_list = [[tuple(v) for v in xyr[ptr[r]:ptr[r + 1]]] for r in range(hole.size)]
    edges = mask_ref.boundary_edges(ring_list)
    n = adj.shape[0]
    rows = np.repeat(np.arange(n), np.diff(adj.indptr))
    within = np.array([mask_ref.segment_within(xy[i], xy[j], edges) for i, j in zip(rows, adj.indices)], dtype=bool)
    gone = within if negative else ~within
    drop = {(int(i), int(j)) for i, j in zip(rows[gone], adj.indices[gone])}
    out = []
    for m, pos in ((adj, None), (dst, drop)):
        r = np.repeat(np.arange(n), np.diff(m.indptr))
        keep = ~gone if pos is None else np.array([(int(i), int(j)) not in pos for i, j in zip(r, m.indices)], dtype=bool)
        keep &= m.data != 0
        ip = np.r_[0, np.cumsum(np.bincount(r[keep], minlength=n))].astype(m.indptr.dtype)
        res = sp.csr_matrix((m.data[keep], m.indices[keep], ip), shape=m.shape)
        res.indptr, res.indices = ip, m.indices[keep].astype(m.indices.dtype)
        out.append(res)
    return tuple(out)


@pytest.fixture
def host_kernel(monkeypatch):
    calls = []

    def fake(adj, dst, xy, rings, negative, *, device=None):
        calls.append(negative)
        return restated(adj, dst, xy, rings, negative)

    monkeypatch.setattr(_mask, "host_mask", fake)
    return calls


def knn_adata(pts, k=3, set_diag=False):
    n = len(pts)
    d = np.linalg.norm(pts[:, None] - pts[None], axis=-1)
    np.fill_diagonal(d, np.inf)
    idx = np.sort(np.argsort(d, axis=1, kind="stable")[:, :k], axis=1)
    rows = np.repeat(np.arange(n), k)
    adj = sp.csr_matrix((np.ones(n * k, np.float32), idx.ravel(), np.arange(0, n * k + 1, k)), shape=(n, n))
    dst = sp.csr_matrix((d[rows, idx.ravel()], idx.ravel().copy(), np.arange(0, n * k + 1, k)), shape=(n, n))
    if set_diag:
        adj.setdiag(1.0)
        dst.setdiag(0.0)
    a = AnnDataLite(shape=(n, 0))
    a.obsm["spatial"] = pts
    a.obsp["spatial_connectivities"] = adj
    a.obsp["spatial_distances"] = dst
    return a


def test_keys_uns_and_copy(host_kernel):
    a = knn_adata(sdata_mask_graph_points())
    adj0, dst0 = a.obsp["spatial_connectivities"].copy(), a.obsp["spatial_distances"].copy()
    assert sq.gr.mask_graph(a, "table", CONCAVE, key_added="mask2") is None
    assert set(a.obsp) >= {"mask2_spatial_connectivities", "mask2_spatial_distances"}
    assert a.uns["mask2_spatial_neighbors"] == {"connectivities_key": "mask2_spatial_connectivities", "distances_key": "mask2_spatial_distances",
                                                "unfiltered_graph_key": "spatial_connectivities",
                                                "params": {"negative_mask": False, "table_key": "table"}}
    pos = a.obsp["mask2_spatial_connectivities"]
    res = sq.gr.mask_graph(a, "table", CONCAVE, negative_mask=True, copy=True)
    assert isinstance(res, tuple) and len(res) == 2 and "mask_spatial_connectivities" not in a.obsp
    neg = res[0]
    # the reference's identity: positive and negative masks partition the entries; the source graphs are untouched
    assert pos.sum() + neg.sum() == adj0.sum() and pos.multiply(neg).nnz == 0
    assert 0 < pos.nnz < adj0.nnz
    for m0, key in ((adj0, "spatial_connectivities"), (dst0, "spatial_distances")):
        m = a.obsp[key]
        assert (m != m0).nnz == 0 and np.array_equal(m.indptr, m0.indptr) and np.array_equal(m.indices, m0.indices)
    assert host_kernel == [False, True]


def test_zero_elimination_and_diagonal(host_kernel):
    pts = np.array([(1.0, 1.0), (1.0, 1.0), (2.0, 1.0), (3.0, 1.0), (10.0, 10.0)])
    a = knn_adata(pts, k=2, set_diag=True)
    adj, dst = sq.gr.mask_graph(a, None, SQUARE_HOLE, copy=True)
    # kept: the diagonal of the interior points (zero-length, interior) and every edge among points 0..3
    assert adj[4, 4] == 0 and adj[0, 0] == 1 and adj[0, 1] == 1
    assert dst.nnz == np.count_nonzero(dst.data) and (dst.data != 0).all()  # zero distances (diagonal, coincident 0-1) gone
    assert adj.nnz == sum(1 for i, j in zip(*a.obsp["spatial_connectivities"].nonzero()) if i < 4 and j < 4)
    assert adj.dtype == np.float32 and dst.dtype == np.float64 and adj.indices.dtype == a.obsp["spatial_connectivities"].indices.dtype


def test_dst_structure_differs(host_kernel):
    pts = sdata_mask_graph_points()
    a = knn_adata(pts)
    a.obsp["spatial_connectivities"].setdiag(1.0)  # only adj stores the diagonal
    adj, dst = sq.gr.mask_graph(a, "t", CONCAVE, copy=True)
    src = a.obsp["spatial_distances"]
    kept = {(i, j) for i, j in zip(*adj.nonzero())}
    assert {(i, j) for i, j in zip(*dst.nonzero())} == {(i, j) for i, j in zip(*src.nonzero()) if (i, j) in kept}


def test_reference_error_and_refusals(host_kernel):
    a = knn_adata(sdata_mask_graph_points())
    with pytest.raises(ValueError, match="`polygon_mask` should be of type `Polygon` or `MultiPolygon`, got"):
        sq.gr.mask_graph(a, "t", Geo("Point", (0, 1)))
    with pytest.raises(ValueError, match="`polygon_mask` should be of type"):
        sq.gr.mask_graph(a, "t", [(0, 0), (1, 0), (0, 1)])
    b = knn_adata(sdata_mask_graph_points())
    b.obsp["spatial_connectivities"] = b.obsp["spatial_connectivities"].tocsc()
    with pytest.raises(ValueError, match="CSR"):
        sq.gr.mask_graph(b, "t", CONCAVE)
    c = knn_adata(sdata_mask_graph_points())
    m = c.obsp["spatial_distances"]
    m.indices[1] = m.indices[0]  # row 0 stores one column twice
    with pytest.raises(ValueError, match="more than once"):
        sq.gr.mask_graph(c, "t", CONCAVE)
    d = knn_adata(sdata_mask_graph_points())
    d.obsm["spatial"] = np.c_[d.obsm["spatial"], np.zeros(12)]
    with pytest.raises(NotImplementedError):
        sq.gr.mask_graph(d, "t", CONCAVE)
    for bad in (1e37, 1e-40, np.nan):
        e = knn_adata(sdata_mask_graph_points())
        e.obsm["spatial"] = e.obsm["spatial"].copy()
        e.obsm["spatial"][3, 1] = bad
        with pytest.raises(ValueError, match="coordinates"):
            sq.gr.mask_graph(e, "t", CONCAVE)
    with pytest.raises(ValueError, match="Polygon vertices"):
        sq.gr.mask_graph(a, "t", poly([(0, 0), (1e-200, 0), (1, 1)]))
    assert host_kernel == []


def test_table_selection(host_kernel):
    class SData:
        def __init__(self, tables):
            self.tables = tables

    a, b = knn_adata(sdata_mask_graph_points()), knn_adata(sdata_mask_graph_points() + 100)
    sdata = SData({"table": a, "other": b})
    sq.gr.mask_graph(sdata, "other", CONCAVE)
    assert "mask_spatial_connectivities" in b.obsp and "mask_spatial_connectivities" not in a.obsp
    assert b.obsp["mask_spatial_connectivities"].nnz == 0  # far outside the polygon
    assert b.uns["mask_spatial_neighbors"]["params"]["table_key"] == "other"
    with pytest.raises(ValueError, match="not found"):
        sq.gr.mask_graph(sdata, "missing", CONCAVE)
