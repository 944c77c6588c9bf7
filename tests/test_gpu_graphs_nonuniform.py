"""GPU parity of the kNN and radius searches on point sets the uniform cell grid fits badly.

``build_grid`` sizes its cells from the bounding box (kNN: ``sqrt(area * pts_per_cell / n)``, radius: the radius) and
coarsens the grid by 1.5x until it has at most ``4n + 16`` cells.  On clustered tissue with a few outlying spots one cell
holds thousands of points and an outlier's ring search walks far; ``graph_knn_kernel`` stops after ring ``r`` once its
k-th distance is below ``r * cell``.  Indices and distances are compared exactly with scikit-learn (float64
``sqrt(dx*dx + dy*dy)`` without contraction on both sides)."""

from __future__ import annotations

import math

import numpy as np
import pytest
from sklearn.neighbors import NearestNeighbors

from squidpy_b200.gr import GridBuilder, knn_2d, radius_2d

pytestmark = pytest.mark.gpu
KS = (1, 8, 9, 16, 17, 32, 33, 64)  # both ends of every KMAX instance (8, 16, 32, 64)


def nn(**kw) -> NearestNeighbors:
    """scikit-learn's kd_tree, whose distance arithmetic the kernels reproduce; ``algorithm='auto'`` switches to the
    brute-force dot-product distances when k >= n / 2, which round differently."""
    return NearestNeighbors(algorithm="kd_tree", **kw)


def knn_grid(xy: np.ndarray, k: int) -> tuple[float, int, int]:
    """(cell, gx, gy) of ``sqb_knn_2d``: ``build_grid(..., cell_hint = 0, pts_per_cell = k <= 8 ? 2.5 : k / 3.0)``."""
    return grid_geometry(xy, 0.0, 2.5 if k <= 8 else k / 3.0)


def grid_geometry(xy: np.ndarray, cell_hint: float, pts_per_cell: float) -> tuple[float, int, int]:
    """graph.cu ``build_grid``: ``cell = cell_hint`` or ``sqrt(area * pts_per_cell / n)``, then ``cell *= 1.5`` while
    ``gx * gy > 4n + 16`` with ``gx = floor(w / cell) + 1``."""
    n = xy.shape[0]
    w, h = np.ptp(xy[:, 0]), np.ptp(xy[:, 1])
    cell = cell_hint
    if not cell > 0.0:
        cell = math.sqrt((w if w > 0 else 1.0) * (h if h > 0 else 1.0) * pts_per_cell / n)
    while (math.floor(w / cell) + 1.0) * (math.floor(h / cell) + 1.0) > 4.0 * n + 16.0:
        cell *= 1.5
    return cell, int(math.floor(w / cell) + 1), int(math.floor(h / cell) + 1)


def _blobs(shift: float = 0.0) -> np.ndarray:
    rng = np.random.default_rng(42)
    centres = rng.uniform(2e4, 8e4, (3, 2))
    pts = [c + rng.normal(0.0, 1.0, (15000, 2)) for c in centres]
    pts.append(rng.uniform(0.0, 1e5, (40, 2)))  # outliers spread over the whole box
    return np.concatenate(pts) + shift


@pytest.fixture(scope="module", params=[0.0, 1e9], ids=["origin", "shifted_1e9"])
def blobs(request):
    """Three sigma = 1 blobs of 15 000 points and 40 uniform outliers in a 1e5 box (optionally shifted by 1e9, where the
    cell coordinate (v - x0) * inv_cell rounds), with scikit-learn's 65 nearest neighbours of every point."""
    xy = _blobs(request.param)
    d_ref, i_ref = nn(n_neighbors=max(KS) + 1).fit(xy).kneighbors()
    for k in KS:  # the k-th neighbour is unique: the k nearest form a well-defined set
        assert (d_ref[:, k - 1] < d_ref[:, k]).all(), k
    return xy, d_ref, i_ref


@pytest.mark.parametrize("k", KS)
def test_knn_blobs_with_outliers(blobs, k):
    xy, d_ref, i_ref = blobs
    cell, gx, gy = knn_grid(xy, k)
    in_cell = np.bincount(np.floor((xy[:, 0] - xy[:, 0].min()) / cell).astype(np.int64) * gy
                          + np.floor((xy[:, 1] - xy[:, 1].min()) / cell).astype(np.int64))
    assert in_cell.max() > 10000  # a whole blob in one or a few cells
    far = np.ceil(d_ref[-40:, k - 1] / cell)
    assert far.max() > 16  # some outlier walks more than 16 rings before its k-th neighbour is certain
    dist, idx = knn_2d(xy, k)
    order = np.argsort(i_ref[:, :k], axis=1)
    np.testing.assert_array_equal(idx, np.take_along_axis(i_ref[:, :k], order, 1))
    np.testing.assert_array_equal(dist, np.take_along_axis(d_ref[:, :k], order, 1))


def test_knn_every_other_point():
    rng = np.random.default_rng(9)
    xy = rng.random((65, 2)) * [1e3, 1.0]
    dist, idx = knn_2d(xy, 64)
    np.testing.assert_array_equal(idx, np.array([np.delete(np.arange(65), i) for i in range(65)]))
    d2 = ((xy[:, None, :] - xy[None, :, :]) ** 2).sum(-1)
    exp = np.sqrt(np.array([np.delete(d2[i], i) for i in range(65)]))
    d_ref, i_ref = nn(n_neighbors=64).fit(xy).kneighbors()
    np.testing.assert_array_equal(dist, np.take_along_axis(d_ref, np.argsort(i_ref, axis=1), 1))
    np.testing.assert_allclose(dist, exp, rtol=1e-15)
    with pytest.raises(NotImplementedError, match=r"n_neighbors=65 outside \[1, 64\]"):
        knn_2d(xy, 65)
    with pytest.raises(ValueError, match="n_neighbors <= n_samples_fit"):
        knn_2d(xy[:64], 64)


def _check_radius(xy, radius):
    indptr, idx, dist = radius_2d(xy, radius)
    d_ref, i_ref = nn(radius=radius).fit(xy).radius_neighbors()
    np.testing.assert_array_equal(np.diff(indptr), [len(r) for r in i_ref])
    for r in range(xy.shape[0]):
        o = np.argsort(i_ref[r])
        np.testing.assert_array_equal(idx[indptr[r] : indptr[r + 1]], i_ref[r][o])
        np.testing.assert_array_equal(dist[indptr[r] : indptr[r + 1]], d_ref[r][o])
    return np.diff(indptr)


def test_radius_far_below_the_spacing_coarsens_the_grid():
    """A 1e6-wide extent searched with radius 1: cells of edge 1 would be 1e12, so the 4n + 16 cap coarsens the grid."""
    rng = np.random.default_rng(1)
    base = rng.uniform(0.0, 1e6, (10000, 2))
    near = base[:3000] + rng.uniform(-0.7, 0.7, (3000, 2))  # partners within radius 1 of some points
    xy = np.concatenate([base, near])
    cell, gx, gy = grid_geometry(xy, 1.0, 2.5)
    assert cell > 1000.0 and gx * gy <= 4 * xy.shape[0] + 16
    cnt = _check_radius(xy, 1.0)
    assert 1000 < (cnt > 0).sum() < xy.shape[0]


def test_radius_with_hundreds_of_neighbours():
    """A large radius: the cell edge equals the radius (the search reaches ceil(1 + 1e-12) = 2 cells on every side) and
    rows hold hundreds of neighbours."""
    rng = np.random.default_rng(2)
    xy = np.concatenate([rng.uniform(0.0, 1000.0, (6000, 2)), rng.normal(500.0, 20.0, (1000, 2))])
    cell, gx, gy = grid_geometry(xy, 120.0, 2.5)
    assert cell == 120.0
    cnt = _check_radius(xy, 120.0)
    assert cnt.max() > 500 and cnt.min() > 10


def test_radius_zero_on_duplicated_points():
    rng = np.random.default_rng(3)
    xy = np.repeat(rng.uniform(0.0, 500.0, (800, 2)), [1, 2, 3, 4] * 200, axis=0)
    cnt = _check_radius(xy, 0.0)
    np.testing.assert_array_equal(cnt, np.repeat([0, 1, 2, 3] * 200, [1, 2, 3, 4] * 200))


@pytest.mark.parametrize("n,k", [(1001, 5), (1000, 5), (2001, 6)])
def test_grid_builder_median_cut(n, k):
    """``GridBuilder``: ``dist < 1.3 * np.median(dist)`` over all n * k candidate distances; n * k odd takes the middle
    value, even the mean of the two middle ones."""
    rng = np.random.default_rng(n)
    xy = rng.random((n, 2)) * 100.0
    d_ref, i_ref = nn(n_neighbors=k).fit(xy).kneighbors()
    med = np.median(d_ref)
    dist, idx, got_med = knn_2d(xy, k, median=True)
    assert got_med == med
    adj, dst = GridBuilder(n_neighs=k).build(xy)
    keep = d_ref < 1.3 * med
    rows = np.repeat(np.arange(n), k)[keep.ravel()]
    exp = np.zeros((n, n), np.float32)
    exp[rows, i_ref.ravel()[keep.ravel()]] = 1.0
    np.testing.assert_array_equal(adj.toarray(), exp)
    assert 0 < (~keep).sum()  # the cut removes some candidates
