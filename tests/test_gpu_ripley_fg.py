"""GPU parity of ripley F / G: ``nn_distance_hist`` against the CPU restatement (scikit-learn's KDTree + np.histogram),
exact integer bin counts, and ``ripley`` against the reference's golden output and against its own host path."""

from __future__ import annotations

import os
import warnings

import numpy as np
import pytest

import squidpy_b200 as sq
from squidpy_b200.gr import _ripley, nn_distance_hist
from tests import nndist_ref
from tests.golden.make_golden_ripley_fg import CASES, N_SIM, SEED, make_adata
from tools import synth

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ripley_fg.npz")
NN_SHARED_BINS = 8192  # graph.cu: histograms of up to this many bins are kept in shared memory


def _check(pool, tasks, support, n_rows):
    exp = nndist_ref.eval_tasks(pool, tasks, support, n_rows)
    got = nn_distance_hist(pool, tasks, support, n_rows)
    np.testing.assert_array_equal(got, exp)
    parts = [nn_distance_hist(pool, tasks, support, n_rows, shard=(r, 3)) for r in range(3)]
    np.testing.assert_array_equal(sum(parts), exp)  # query-block shards add up (multi-GPU path)
    return exp


@pytest.mark.parametrize("k", [1, 2, 8, 33, 64])
def test_vs_restatement_random_and_far_queries(k):
    rng = np.random.default_rng(k)
    ref_a = rng.random((3000, 2)) * 100.0
    ref_b = rng.random((500, 2)) * 10.0 + 400.0  # a small set far from everything
    qry = np.concatenate([rng.random((2500, 2)) * 100.0, rng.random((700, 2)) * 2000.0 - 800.0])  # many far outside both boxes
    pool = np.concatenate([ref_a, ref_b, qry])
    q0 = 3500
    tasks = np.array([[0, 3000, q0, pool.shape[0], k, 0], [3000, 3500, q0, pool.shape[0], k, 1], [3000, 3500, 0, 3000, k, 1],
                      [0, 3000, q0, q0, k, 2]])  # the last: an empty query range
    support = np.linspace(0, 900.0, 50)
    exp = _check(pool, tasks, support, 3)
    assert exp[0].sum() > 0 and exp[1].sum() > 0 and (exp[2] == 0).all()


@pytest.mark.parametrize("k", [1, 2, 8, 33, 64])
def test_lattice_ties_and_exact_edges(k):
    gx, gy = np.meshgrid(np.arange(40), np.arange(40))
    lat = np.stack([gx.ravel(), gy.ravel()], 1).astype(np.float64)
    off = lat[(lat[:, 0] % 3 == 0) & (lat[:, 1] % 2 == 0)] + np.array([100.0, -50.0])  # a shifted sub-lattice, far away
    pool = np.concatenate([lat, off, lat])
    n = lat.shape[0]
    tasks = np.array([[0, n, n + off.shape[0], pool.shape[0], k, 0], [0, n, n, n + off.shape[0], k, 1]])
    support = np.arange(0.0, 13.0)  # integer edges: distances 1, 2, 3 ... sit exactly on them; larger ones dropped
    exp = _check(pool, tasks, support, 2)
    assert exp[0].sum() > 0 and exp[0, 0] > 0  # zero distances (the query set repeats the reference) count


@pytest.mark.parametrize("S,shared", [(NN_SHARED_BINS + 1, True), (NN_SHARED_BINS + 2, False), (20000, False)])
def test_histogram_branches(S, shared):
    assert (S - 1 <= NN_SHARED_BINS) == shared
    rng = np.random.default_rng(S)
    pool = rng.random((6000, 2)) * 50.0
    tasks = np.array([[0, 2000, 2000, 6000, 2, 0], [2000, 2100, 0, 6000, 1, 1]])
    support = np.sort(rng.random(S)) * 4.0
    support[3] = support[2]  # a repeated edge
    exp = _check(pool, tasks, support, 2)
    assert exp.sum() > 0


def test_repeated_edges_and_max_dist_zero():
    rng = np.random.default_rng(5)
    pool = np.concatenate([rng.integers(0, 30, (800, 2)).astype(np.float64)] * 2)
    tasks = np.array([[0, 800, 800, 1600, 3, 0]])
    exp = _check(pool, tasks, np.zeros(5), 1)
    assert exp[0, -1] > 0 and (exp[0, :-1] == 0).all()  # only exact zeros, all in the closed last bin


def test_invalid_tasks_are_refused():
    pool = np.random.default_rng(0).random((10, 2))
    with pytest.raises(ValueError, match="n_neighbors"):
        nn_distance_hist(pool, np.array([[0, 3, 3, 10, 4, 0]]), np.linspace(0, 1, 5), 1)
    with pytest.raises(NotImplementedError):
        nn_distance_hist(pool, np.array([[0, 10, 0, 10, 65, 0]]), np.linspace(0, 1, 5), 1)
    with pytest.raises(ValueError, match="ascending"):
        nn_distance_hist(pool, np.array([[0, 10, 0, 10, 1, 0]]), np.array([0.0, 2.0, 1.0]), 1)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_api_ripley_fg_golden(case):
    g = np.load(GOLDEN)
    mode, metric, n_steps, max_dist, n_obs = CASES[case]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        res = sq.gr.ripley(make_adata(g["xy"], g["codes"]), "cluster", mode=mode, metric=metric, n_neigh=2, n_simulations=N_SIM,
                           n_observations=n_obs, max_dist=max_dist, n_steps=n_steps, seed=SEED, copy=True)
    np.testing.assert_array_equal(res["bins"], g[f"c{case}_bins"])
    np.testing.assert_array_equal(res[f"{mode}_stat"]["stats"].to_numpy(), g[f"c{case}_stat"])
    np.testing.assert_array_equal(res["sims_stat"]["stats"].to_numpy(), g[f"c{case}_sims"])
    np.testing.assert_array_equal(res["pvalues"], g[f"c{case}_pvalues"])


def _host_only(monkeypatch):
    """Route every set to scikit-learn (the host path of non-kd_tree sets)."""
    monkeypatch.setattr(_ripley, "_kd_tree_euclidean", lambda metric, n_neigh, n_fit: False)


def _region_labels(pts, n):
    """Clusters as spatial blocks: vertical strips of equal width."""
    x = pts[:, 0]
    return np.minimum(((x - x.min()) / (np.ptp(x) + 1e-9) * n).astype(int), n - 1)


@pytest.mark.parametrize("labels", ["random", "region"])
@pytest.mark.parametrize("mode", ["G", "F"])
def test_configs4_device_equals_host(monkeypatch, labels, mode):
    import pandas as pd

    pts = synth.thomas_points(300_000, seed=5)
    if labels == "random":
        lab = synth.dirichlet_labels(300_000, 12, seed=5)
    else:
        lab = pd.Series(pd.Categorical.from_codes(_region_labels(pts, 12), categories=[f"r{i:02d}" for i in range(12)]))
    ad = synth.make_adata(pts, None, lab)
    kw = dict(mode=mode, n_simulations=5, n_observations=1000, seed=3, copy=True)
    dev = sq.gr.ripley(ad, "cluster", **kw)
    with monkeypatch.context() as m:
        _host_only(m)
        host = sq.gr.ripley(ad, "cluster", **kw)
    for key in (f"{mode}_stat", "sims_stat"):
        assert dev[key].equals(host[key])
    np.testing.assert_array_equal(dev["pvalues"], host["pvalues"])
