"""Ripley's L for every ``KDTree`` metric, checked without a GPU: the pair-count restatement (``tests/pairs_ref.py``) against
scikit-learn's ``two_point_correlation`` for all nine names on inputs full of exact ties, and the public ``ripley(mode="L")``
(with ``pair_counts`` replaced by that restatement) against the unmodified reference's golden output."""

from __future__ import annotations

import os

import numpy as np
import pytest

import squidpy_b200 as sq
from squidpy_b200.gr import _ripley
from tests import pairs_ref
from tests.golden.make_golden_ripley_l_metrics import CASES, METRICS, N_SIM, SEED, make_adata

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ripley_l_metrics.npz")
CODE = {name: code for code, names in pairs_ref.NAMES.items() for name in names}


def _lattice(side, scale=1.0, offset=0.0):
    gx, gy = np.meshgrid(np.arange(side, dtype=np.float64), np.arange(side, dtype=np.float64))
    return np.stack([gx.ravel(), gy.ravel()], 1) * scale + offset


def _tie_support(points, metric, n, seed):
    """``n`` distances that occur between points of ``points`` (computed with the metric's own float64 arithmetic, so pairs
    lie exactly on every radius), their float64 neighbours on both sides, a repeated radius, 0, -0.0 and a negative one."""
    rng = np.random.default_rng(seed)
    p = points[rng.choice(points.shape[0], min(400, points.shape[0]), replace=False)]
    d = np.unique(pairs_ref.pair_dist(p[:, None, 0] - p[None, :, 0], p[:, None, 1] - p[None, :, 1], metric))
    on = rng.choice(d, min(n, d.size), replace=False)
    sup = np.concatenate([on, np.nextafter(on, -np.inf), np.nextafter(on, np.inf), on[:3], [0.0, -0.0, -1.0]])
    return np.sort(sup)


def _inputs():
    rng = np.random.default_rng(5)
    yield "random", rng.random((3000, 2)) * 1000, None
    yield "lattice40", _lattice(40), None
    yield "lattice30x0.1+3", _lattice(30, 0.1, 3.0), None
    yield "offset1e9", rng.random((1500, 2)) * 100 + 1e9, None


@pytest.mark.parametrize("name", METRICS)
def test_restatement_matches_two_point_correlation(name):
    from sklearn.neighbors import KDTree

    code = CODE[name]
    for label, pts, _ in _inputs():
        sup = _tie_support(pts, code, 40, seed=len(label))
        exp = pairs_ref.pair_counts(pts, sup, code)
        assert (np.diff(exp) > 0).sum() >= 20, label  # the ties move the counts
        tree = KDTree(pts, metric=name)
        np.testing.assert_array_equal(tree.two_point_correlation(pts, sup, dualtree=True), exp, err_msg=f"{label} dualtree")
        np.testing.assert_array_equal(tree.two_point_correlation(pts, sup, dualtree=False), exp, err_msg=f"{label} single")


def test_strict_comparison_would_differ():
    """The lattice supports discriminate ``<=`` from ``<`` in every metric class."""
    pts = _lattice(30, 0.1, 3.0)
    for code in (0, 1, 2):
        sup = _tie_support(pts, code, 40, seed=1)
        le = pairs_ref.pair_counts(pts, sup, code)
        lt = pairs_ref.pair_counts(pts, np.nextafter(sup, -np.inf), code)
        assert (le != lt).sum() >= 20, code


def test_metric_code_importable_from_both_modules():
    from squidpy_b200._metrics import metric_code
    from squidpy_b200.tl import _var_by_distance

    assert _var_by_distance.metric_code is metric_code
    for name in METRICS:
        assert metric_code(name) == CODE[name]
        assert _ripley._check_l_metric(name) == CODE[name]


@pytest.fixture()
def host_kernel(monkeypatch):
    """``pair_counts`` replaced by the CPU restatement (and no CUDA context): every metric code the device would get."""
    calls = []

    def fake(groups, support, *, metric=0, ctx=None, shard=(0, 1)):
        calls.append(metric)
        return pairs_ref.group_counts(groups, support, metric)

    monkeypatch.setattr(_ripley, "pair_counts", fake)
    monkeypatch.setattr(_ripley, "default_context", lambda device=None: None)
    return calls


@pytest.mark.parametrize("case", range(len(CASES)))
def test_ripley_l_reproduces_reference_golden(host_kernel, case):
    g = np.load(GOLDEN)
    metric, n_steps, max_dist, n_obs = CASES[case]
    res = sq.gr.ripley(make_adata(g["xy"], g["codes"]), "cluster", mode="L", metric=metric, n_simulations=N_SIM, n_observations=n_obs,
                       max_dist=max_dist, n_steps=n_steps, seed=SEED, copy=True)
    np.testing.assert_array_equal(res["bins"], g[f"c{case}_bins"])
    np.testing.assert_array_equal(res["L_stat"]["stats"].to_numpy(), g[f"c{case}_stat"])
    np.testing.assert_array_equal(res["sims_stat"]["stats"].to_numpy(), g[f"c{case}_sims"])
    np.testing.assert_array_equal(res["pvalues"], g[f"c{case}_pvalues"])
    assert host_kernel == [CODE[metric]]  # one device call per ripley(), with the metric's kernel code


def test_golden_discriminates_the_metric_classes():
    """The three classes give different statistics on every fixture with a positive ``max_dist``; the four euclidean names,
    the three manhattan names and the two chebyshev names agree exactly."""
    g = np.load(GOLDEN)
    for shape in {c[1:] for c in CASES}:
        by_name = {m: g[f"c{CASES.index((m, *shape))}_stat"] for m in METRICS}
        for code, names in pairs_ref.NAMES.items():
            for name in names[1:]:
                np.testing.assert_array_equal(by_name[name], by_name[names[0]])
        if shape[1] != 0.0:
            stats = [by_name[names[0]] for names in pairs_ref.NAMES.values()]
            assert not np.array_equal(stats[0], stats[1]) and not np.array_equal(stats[0], stats[2]) and not np.array_equal(stats[1], stats[2])


def test_single_point_cluster_in_golden():
    g = np.load(GOLDEN)
    assert (np.bincount(g["codes"]) == 1).any()


def test_unsupported_metric_keeps_reference_error(host_kernel):
    g = np.load(GOLDEN)
    with pytest.raises(ValueError, match=r"Unsupported metric 'cosine'\. Ripley's L supports \["):
        sq.gr.ripley(make_adata(g["xy"], g["codes"]), "cluster", mode="L", metric="cosine", n_simulations=2, copy=True)
    assert host_kernel == []
