"""GPU parity of tl.var_by_distance: ``nn_min_dist`` against scikit-learn's ``KDTree.query`` (bit for bit, every metric name)
on inputs that stress the hierarchy, the four anchor geometries at 1 M queries, and ``var_by_distance`` against the
reference's golden frames and against itself with the kernel replaced by the scikit-learn restatement."""

from __future__ import annotations

import os

import numpy as np
import pandas as pd
import pytest

import squidpy_b200 as sq
from squidpy_b200 import AnnDataLite
from squidpy_b200.tl import _var_by_distance, nn_min_dist
from squidpy_b200.tl._var_by_distance import metric_code
from tests import nearest_ref
from tests.golden.make_golden_var_by_distance import CASES, decode, groups_arg, make_adata
from tools import var_by_distance_time as vt

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "var_by_distance.npz")
NAMES = ["euclidean", "l2", "minkowski", "p", "manhattan", "cityblock", "l1", "chebyshev", "infinity"]
LEAF = 16  # nearest.cu: points per leaf


def _kdtree(ref, qry, name):
    from sklearn.metrics import DistanceMetric
    from sklearn.neighbors import KDTree

    return KDTree(ref, metric=DistanceMetric.get_metric(name)).query(qry)[0][:, 0]


def _check(ref, qry, name):
    pool = np.concatenate([ref, qry])
    tasks = np.array([[0, len(ref), len(ref), len(pool), 0]])
    got = nn_min_dist(pool, tasks, metric_code(name), len(qry))
    np.testing.assert_array_equal(got, _kdtree(ref, qry, name))


def _inputs(seed):
    rng = np.random.default_rng(seed)
    u = rng.random((5000, 2)) * 1000
    lat = np.stack(np.meshgrid(np.arange(40.0), np.arange(30.0)), -1).reshape(-1, 2)
    return {
        "uniform": (u[:3000], u[3000:]),
        "far_queries": (u[:2000], (rng.random((3000, 2)) - 0.5) * 2e6),  # 10^3 x the extent outside the box
        "single_anchor": (u[:1], u[1:]),
        "one_point": (np.repeat(u[:1], 100, axis=0), u[100:]),
        "collinear": (np.stack([u[:700, 0], np.full(700, 500.0)], 1), u[700:]),  # zero-height box
        "lattice": (lat[::3], lat + rng.integers(0, 2, lat.shape) * 0.5),  # many equidistant anchors
        "offset_1e9": (u[:2500] + 1e9, u[2500:] + 1e9),
    }


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("kind", ["uniform", "far_queries", "single_anchor", "one_point", "collinear", "lattice", "offset_1e9"])
def test_kernel_inputs(kind, name):
    ref, qry = _inputs(7)[kind]
    _check(ref, qry, name)


@pytest.mark.parametrize("name", ["euclidean", "manhattan", "chebyshev"])
@pytest.mark.parametrize("m", [LEAF - 1, LEAF, LEAF + 1, 2 * LEAF + 1, (1 << 20) + 1])
def test_set_sizes(m, name):
    rng = np.random.default_rng(m)
    ref = rng.random((m, 2)) * 100
    qry = rng.random((20000, 2)) * 120 - 10
    _check(ref, qry, name)


def test_tasks_share_query_range_and_leave_gaps_nan():
    rng = np.random.default_rng(3)
    pool = rng.random((6000, 2)) * 500
    tasks = np.array([[0, 100, 1000, 6000, 10], [100, 1000, 1000, 6000, 5020], [4000, 4001, 1000, 6000, 10030],
                      [0, 100, 50, 50, 16100],  # an empty query range
                      [2000, 2500, 0, 1000, 15030]])
    for code in range(3):
        got = nn_min_dist(pool, tasks, code, 16100)
        np.testing.assert_array_equal(got, nearest_ref.eval_tasks(pool, tasks, code, 16100))
        written = np.zeros(16100, dtype=bool)
        for _, _, qb, qe, ob in tasks:
            written[ob : ob + qe - qb] = True
        assert np.isfinite(got[written]).all() and np.isnan(got[~written]).all() and (~written).sum() == 10 + 10 + 10 + 70


@pytest.mark.parametrize("pool, tasks, metric, n_out, match", [
    (np.array([[0.0, np.nan], [1.0, 1.0]]), [[0, 1, 1, 2, 0]], 0, 1, "not finite"),
    (np.array([[0.0, np.inf], [1.0, 1.0]]), [[1, 2, 0, 2, 0]], 0, 2, "not finite"),
    (np.zeros((4, 2)), [[1, 1, 0, 4, 0]], 0, 4, "empty reference"),
    (np.zeros((4, 2)), [[0, 5, 0, 4, 0]], 0, 4, "outside"),
    (np.zeros((4, 2)), [[0, 2, 2, 5, 0]], 0, 4, "outside"),
    (np.zeros((4, 2)), [[0, 2, 0, 4, 1]], 0, 4, "writes outside"),
    (np.zeros((4, 2)), [[0, 2, 0, 4, -1]], 0, 8, "writes outside"),
    (np.zeros((4, 2)), [[0, 2, 0, 4, 0], [0, 1, 0, 4, 3]], 0, 8, "overlap"),
    (np.zeros((4, 2)), [[0, 2, 0, 4, 0]], 3, 4, "metric"),
])
def test_validation_errors(pool, tasks, metric, n_out, match):
    with pytest.raises(ValueError, match=match):
        nn_min_dist(pool, np.array(tasks), metric, n_out)


@pytest.mark.parametrize("name", vt.GEOMETRIES + ("corner",))
def test_geometries_at_1m_queries(name):
    xy, mask = vt.geometry(name, 1_000_000, seed=5)
    _check(xy[mask], xy, "euclidean")


@pytest.mark.parametrize("case", range(len(CASES)))
def test_frame_equals_reference_golden(case):
    g = np.load(GOLDEN)
    groups, kw = CASES[case]
    df = sq.tl.var_by_distance(make_adata(AnnDataLite), groups_arg(groups), copy=True, **kw)
    pd.testing.assert_frame_equal(df, decode(g, f"case{case}"), check_exact=True)


def _restated(monkeypatch):
    monkeypatch.setattr(_var_by_distance, "nn_min_dist", lambda p, t, m, n, *, ctx=None: nearest_ref.eval_tasks(p, t, m, n))


@pytest.mark.parametrize("metric", ["euclidean", "manhattan", "chebyshev"])
def test_1m_cells_4_slides_3_anchors_vs_restatement(monkeypatch, metric):
    adata = vt.make_adata("lines", 1_000_000)
    got = sq.tl.var_by_distance(adata, vt.GROUPS, metric=metric, **vt.KW)
    _restated(monkeypatch)
    exp = sq.tl.var_by_distance(adata, vt.GROUPS, metric=metric, **vt.KW)
    pd.testing.assert_frame_equal(got, exp, check_exact=True)


def test_torch_cuda_coordinates_give_the_host_frame():
    import torch

    adata = vt.make_adata("disc", 200_000)
    exp = sq.tl.var_by_distance(adata, vt.GROUPS, **vt.KW)
    adata.obsm["spatial"] = torch.from_numpy(adata.obsm["spatial"]).cuda()
    got = sq.tl.var_by_distance(adata, vt.GROUPS, **vt.KW)
    pd.testing.assert_frame_equal(got, exp, check_exact=True)
