"""GPU pair counts for the manhattan and chebyshev metrics (``pair_counts(..., metric=1 / 2)``) and the public
``ripley(mode="L")`` for all nine ``KDTree`` metric names.  The counts are integers: every comparison, with the numpy
restatement (``tests/pairs_ref.py``), scikit-learn's ``two_point_correlation`` and the reference's golden output, is exact."""

from __future__ import annotations

import os

import numpy as np
import pytest

import squidpy_b200 as sq
from squidpy_b200.gr import pair_counts
from tests import pairs_ref
from tests.device_attrs import H100_SMEM_OPTIN, smem_optin
from tests.golden.make_golden_ripley_l_metrics import CASES, N_SIM, SEED, make_adata
from tests.test_gpu_pairs_shared_hist import lane_private
from tests.test_ripley_l_metrics_host import CODE, _lattice, _tie_support
from tools import synth

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ripley_l_metrics.npz")


@pytest.fixture(scope="module")
def optin():
    return smem_optin()


def _variant(S, optin, expect_lanepriv, near_boundary):
    """Skip a case that straddles the boundary on a device with another opt-in limit; otherwise assert the branch it takes."""
    if near_boundary and optin != H100_SMEM_OPTIN:
        pytest.skip(f"boundary case written for {H100_SMEM_OPTIN} B of opt-in shared memory per block, this device has {optin} B")
    assert lane_private(S, 8, optin) == expect_lanepriv, (S, optin)


def _kdtree(groups, sup, metric):
    from sklearn.neighbors import KDTree

    return np.stack([KDTree(g, metric=pairs_ref.METRICS[metric]).two_point_correlation(g, sup, dualtree=True) if len(g)
                     else np.zeros(sup.size, np.int64) for g in groups])


@pytest.mark.parametrize("metric", [1, 2])
def test_edge_inputs_match_restatement_and_sklearn(metric):
    rng = np.random.default_rng(metric)
    lat = _lattice(30, 0.1, 3.0)
    groups = [rng.random((1500, 2)) * 500, np.zeros((0, 2)), np.array([[2.5, -7.0]]), lat, rng.random((1023, 2)) * 60 + 1e9,
              rng.random((1024, 2)) * 200, rng.integers(0, 25, (1025, 2)).astype(np.float64)]
    sup = _tie_support(lat, metric, 60, seed=metric)  # lattice distances, their neighbours, repeats, 0, -0.0 and -1
    assert (sup < 0).any() and (sup == 0).sum() >= 2 and (np.diff(sup) == 0).any()
    exp = pairs_ref.group_counts(groups, sup, metric)
    np.testing.assert_array_equal(exp, _kdtree(groups, sup, metric))
    assert (np.diff(exp[3]) > 0).sum() >= 30  # the lattice has pairs exactly on the radii
    got = pair_counts(groups, sup, metric=metric)
    np.testing.assert_array_equal(got, exp)
    np.testing.assert_array_equal(got[:, sup < 0], 0)  # a negative radius counts nothing, not even self pairs
    np.testing.assert_array_equal(got[1], 0)
    np.testing.assert_array_equal(got[2], np.where(sup >= 0, 1, 0))
    parts = [pair_counts(groups, sup, metric=metric, shard=(r, 3)) for r in range(3)]
    np.testing.assert_array_equal(sum(parts), exp)  # tile shards add up (multi-GPU path)


@pytest.mark.parametrize("metric", [1, 2])
@pytest.mark.parametrize("S,lanepriv,near", [(204, True, True), (205, False, True), (400, False, False), (4096, False, False)])
def test_histogram_variants_and_tile_edges(optin, metric, S, lanepriv, near):
    _variant(S, optin, lanepriv, near)
    rng = np.random.default_rng(S + metric)
    groups = [rng.random((m, 2)) * 400 for m in (1023, 0, 1, 1024, 1025, 2100)]
    sup = np.sort(rng.random(S) * 350)
    sup[5] = sup[4]
    sup[-1] = 800.0  # holds every pair in both metrics
    exp = pairs_ref.group_counts(groups, sup, metric)
    np.testing.assert_array_equal(exp[:, -1], np.array([len(g) for g in groups]) ** 2)
    assert (exp[:, -1] > exp[:, -2]).any()  # the last radius adds pairs: a dropped last bin would show
    np.testing.assert_array_equal(pair_counts(groups, sup, metric=metric), exp)
    np.testing.assert_array_equal(sum(pair_counts(groups, sup, metric=metric, shard=(r, 3)) for r in range(3)), exp)
    lat = _lattice(60)
    lsup = np.arange(S, dtype=np.float64) * (118.0 / S)  # integer and fractional radii: lattice pairs lie on the integer ones
    lexp = pairs_ref.pair_counts(lat, lsup, metric)
    np.testing.assert_array_equal(pair_counts([lat], lsup, metric=metric)[0], lexp)


@pytest.mark.parametrize("metric", [1, 2])
def test_infinite_radius_counts_every_pair(metric):
    rng = np.random.default_rng(9)
    pts = rng.random((700, 2)) * 100
    sup = np.array([-np.inf, -2.0, 0.0, 10.0, 50.0, np.inf, np.inf])
    exp = pairs_ref.pair_counts(pts, sup, metric)
    assert exp[0] == exp[1] == 0 and exp[-1] == 700**2
    np.testing.assert_array_equal(pair_counts([pts], sup, metric=metric)[0], exp)


def test_largest_support_accepted_and_invalid_arguments_refused():
    rng = np.random.default_rng(3)
    pts = rng.random((500, 2)) * 100
    sup = np.sort(rng.random(4096) * 120.0)
    for metric in (1, 2):
        np.testing.assert_array_equal(pair_counts([pts], sup, metric=metric)[0], pairs_ref.pair_counts(pts, sup, metric))
        with pytest.raises(ValueError, match=r"S=4097 out of range \[1,4096\]"):
            pair_counts([pts], np.sort(rng.random(4097)), metric=metric)
    for bad in (3, -1):
        with pytest.raises(ValueError, match=rf"metric={bad} is not 0"):
            pair_counts([pts], sup[:10], metric=bad)
    np.testing.assert_array_equal(pair_counts([pts], sup[:10], metric=0)[0], pairs_ref.pair_counts(pts, sup[:10], 0))  # still usable


@pytest.mark.parametrize("case", range(len(CASES)))
def test_ripley_l_matches_reference_golden(case):
    g = np.load(GOLDEN)
    metric, n_steps, max_dist, n_obs = CASES[case]
    res = sq.gr.ripley(make_adata(g["xy"], g["codes"]), "cluster", mode="L", metric=metric, n_simulations=N_SIM, n_observations=n_obs,
                       max_dist=max_dist, n_steps=n_steps, seed=SEED, copy=True)
    np.testing.assert_array_equal(res["bins"], g[f"c{case}_bins"])
    np.testing.assert_array_equal(res["L_stat"]["stats"].to_numpy(), g[f"c{case}_stat"])
    np.testing.assert_array_equal(res["sims_stat"]["stats"].to_numpy(), g[f"c{case}_sims"])
    np.testing.assert_array_equal(res["pvalues"], g[f"c{case}_pvalues"])


def test_euclidean_aliases_are_bit_identical():
    rng = np.random.default_rng(4)
    n = 6000
    ad = synth.make_adata(rng.random((n, 2)) * 3000, None, synth.categorical_labels(n, 6, seed=4))
    runs = {m: sq.gr.ripley(ad, "cluster", mode="L", metric=m, n_simulations=20, n_observations=800, seed=3, copy=True)
            for m in ("euclidean", "l2", "minkowski", "p", "manhattan", "chebyshev")}
    for m in ("l2", "minkowski", "p"):
        for key in ("L_stat", "sims_stat"):
            np.testing.assert_array_equal(runs[m][key]["stats"].to_numpy(), runs["euclidean"][key]["stats"].to_numpy())
        np.testing.assert_array_equal(runs[m]["pvalues"], runs["euclidean"]["pvalues"])
    for m in ("manhattan", "chebyshev"):  # the other classes do change the statistic
        assert not np.array_equal(runs[m]["L_stat"]["stats"].to_numpy(), runs["euclidean"]["L_stat"]["stats"].to_numpy())
