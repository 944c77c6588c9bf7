"""Host logic of ripley F / G on the GPU, checked without a GPU: which reference sets go to the device (scikit-learn's
kd_tree rule), the pool and task list (evaluated here with the CPU restatement instead of the kernel) against the
reference's golden output, and the kernel's binning on squared distances against ``np.histogram``."""

from __future__ import annotations

import os
import warnings

import numpy as np
import pytest

import squidpy_b200 as sq
from squidpy_b200.gr import _ripley
from tests import nndist_ref
from tests.golden.make_golden_ripley_fg import CASES, N_SIM, SEED, make_adata

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ripley_fg.npz")


@pytest.mark.parametrize("metric", ["euclidean", "l2", "minkowski", "manhattan", "chebyshev"])
def test_dispatch_rule_matches_sklearn_fit_method(metric):
    from sklearn.neighbors import NearestNeighbors

    rng = np.random.default_rng(0)
    for n_fit in range(1, 13):
        x = rng.random((n_fit, 2))
        for k in range(1, 7):
            nn = NearestNeighbors(metric=metric, n_neighbors=k).fit(x)
            kd_euclid = nn._fit_method == "kd_tree" and nn.effective_metric_ in ("euclidean", "l2")
            assert _ripley._kd_tree_euclidean(metric, k, n_fit) == kd_euclid, (metric, n_fit, k, nn._fit_method)
    assert not _ripley._kd_tree_euclidean("euclidean", 65, 1000)  # above the kernel's largest k: host
    assert not _ripley._kd_tree_euclidean("euclidean", 2.0, 1000) and not _ripley._kd_tree_euclidean("euclidean", True, 1000)


@pytest.fixture()
def host_kernel(monkeypatch):
    """``nn_distance_hist`` replaced by the CPU restatement (and no CUDA context): every task list the device would get."""
    calls = []

    def fake(points, tasks, support, n_rows, *, ctx=None, shard=(0, 1)):
        calls.append(np.asarray(tasks).copy())
        return nndist_ref.eval_tasks(np.asarray(points), tasks, support, n_rows)

    monkeypatch.setattr(_ripley, "nn_distance_hist", fake)
    monkeypatch.setattr(_ripley, "default_context", lambda device=None: None)
    return calls


@pytest.mark.parametrize("case", range(len(CASES)))
def test_task_list_reproduces_reference_golden(host_kernel, case):
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
    # one device call per ripley(); the 5-point cluster (row 2) is brute force in scikit-learn and never on the device
    assert len(host_kernel) == 1
    rows = set(host_kernel[0][:, 5].tolist())
    assert 2 not in rows and {0, 1, 3} <= rows
    assert any(r >= 4 for r in rows) == (n_obs // 2 > 2)  # simulations of 4 points are brute force too
    if mode == "G":  # cluster c against the points on either side of it in the cluster-sorted pool
        t0 = host_kernel[0][host_kernel[0][:, 5] == 0]
        assert t0.shape[0] == 1 and t0[0, 2] == t0[0, 1] and t0[0, 3] == len(g["codes"])
        t1 = host_kernel[0][host_kernel[0][:, 5] == 1]
        assert t1.shape[0] == 2 and t1[0, 2] == 0 and t1[0, 3] == t1[0, 0] and t1[1, 2] == t1[0, 1]
    else:  # every simulation queries the last cluster's draw
        sims = host_kernel[0][host_kernel[0][:, 5] >= 4]
        last = host_kernel[0][host_kernel[0][:, 5] == 3][0]
        assert (sims[:, 2] == last[2]).all() and (sims[:, 3] == last[3]).all() and (sims[:, 4] == 1).all()


def test_non_euclidean_metric_never_calls_the_device(host_kernel):
    g = np.load(GOLDEN)
    sq.gr.ripley(make_adata(g["xy"], g["codes"]), "cluster", mode="G", metric="manhattan", n_simulations=3, n_observations=20, seed=1, copy=True)
    assert host_kernel == []


def test_too_few_points_keep_sklearn_error(host_kernel):
    g = np.load(GOLDEN)
    with pytest.raises(ValueError, match="n_neighbors"):
        sq.gr.ripley(make_adata(g["xy"], g["codes"]), "cluster", mode="G", n_neigh=6, n_simulations=2, n_observations=20, seed=1, copy=True)


@pytest.mark.parametrize("support", [
    np.arange(13, dtype=np.float64),            # integer edges: lattice distances 1, 2, 3 ... fall on them
    np.zeros(5),                                # max_dist = 0: repeated edges
    np.array([0.0, 1.0, 1.0, 1.0, np.sqrt(2.0), 2.0, 2.0]),
    np.linspace(0, 3.3, 2),
    np.array([0.5, np.sqrt(5.0), 3.0]),         # first edge above 0: smaller distances dropped
])
def test_binning_restatement_matches_np_histogram(support):
    i = np.arange(0, 20)
    d2 = np.concatenate([(i[:, None] ** 2 + i[None, :] ** 2).ravel(), [0.0, 2.0, 5.0, 5.0, 9.0, 144.0, 145.0]]).astype(np.float64)
    d2 = np.concatenate([d2, np.nextafter(d2, 0.0), np.nextafter(d2, np.inf)])
    d2 = d2[d2 >= 0]
    exp = np.histogram(np.sqrt(d2), bins=support)[0]
    np.testing.assert_array_equal(nndist_ref.bin_d2(d2, support), exp)
    assert exp.sum() > 0 or support[-1] == 0.0
