"""Host logic of tl.var_by_distance, checked without a GPU: the CPU restatement of the kernel against brute force, the frame
assembly (with the kernel replaced by that restatement) against the reference's golden frames, and the reference's errors."""

from __future__ import annotations

import os

import numpy as np
import pandas as pd
import pytest

import squidpy_b200 as sq
from squidpy_b200 import AnnDataLite
from squidpy_b200.tl import _var_by_distance
from tests import nearest_ref
from tests.golden.make_golden_var_by_distance import CASES, ERRORS, decode, groups_arg, make_adata

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "var_by_distance.npz")
NAMES = {0: ["euclidean", "l2", "minkowski", "p"], 1: ["manhattan", "cityblock", "l1"], 2: ["chebyshev", "infinity"]}


@pytest.mark.parametrize("metric", [0, 1, 2])
def test_restatement_matches_brute_force(metric):
    rng = np.random.default_rng(metric)
    lattice = np.stack(np.meshgrid(np.arange(12.0), np.arange(9.0)), -1).reshape(-1, 2)  # many equidistant anchors
    pool = np.concatenate([rng.random((400, 2)) * 100, lattice, rng.integers(0, 20, (300, 2)).astype(float), [[3.0, 3.0]] * 5])
    tasks = np.array([[0, 400, 400, 508, 0], [400, 508, 0, 400, 108], [508, 808, 0, 813, 508], [808, 813, 400, 508, 1321],
                      [0, 1, 808, 813, 1429]])
    got = nearest_ref.eval_tasks(pool, tasks, metric, 1440)
    for rb, re, qb, qe, ob in tasks:
        np.testing.assert_array_equal(got[ob : ob + qe - qb], nearest_ref.brute_min_dist(pool[rb:re], pool[qb:qe], metric))
    assert np.isnan(got[1434:]).all()


@pytest.mark.parametrize("name", [n for v in NAMES.values() for n in v])
def test_metric_codes(name):
    assert _var_by_distance.metric_code(name) == next(c for c, v in NAMES.items() if name in v)


@pytest.fixture()
def host_kernel(monkeypatch):
    """``nn_min_dist`` replaced by the CPU restatement (and no CUDA context): every call the device would get."""
    calls = []

    def fake(points, tasks, metric, n_out, *, ctx=None):
        calls.append((np.asarray(points).copy(), np.asarray(tasks).copy()))
        return nearest_ref.eval_tasks(points, tasks, metric, n_out)

    monkeypatch.setattr(_var_by_distance, "nn_min_dist", fake)
    monkeypatch.setattr(_var_by_distance, "default_context", lambda device=None: None)
    return calls


@pytest.mark.parametrize("case", range(len(CASES)))
def test_frame_equals_reference_golden(host_kernel, case):
    g = np.load(GOLDEN)
    groups, kw = CASES[case]
    df = sq.tl.var_by_distance(make_adata(AnnDataLite), groups_arg(groups), copy=True, **kw)
    pd.testing.assert_frame_equal(df, decode(g, f"case{case}"), check_exact=True)
    assert len(host_kernel) == 1  # one device call for every (slide, anchor) combination


@pytest.mark.parametrize("case", [2, 6, 16])
def test_copy_false_writes_obsm(host_kernel, case):
    g = np.load(GOLDEN)
    groups, kw = CASES[case]
    adata = make_adata(AnnDataLite)
    assert sq.tl.var_by_distance(adata, groups_arg(groups), design_matrix_key="dm", **kw) is None
    pd.testing.assert_frame_equal(adata.obsm["dm"], decode(g, f"case{case}"), check_exact=True)


@pytest.mark.parametrize("case", range(len(ERRORS)))
def test_errors_raise_reference_type(host_kernel, case):
    g = np.load(GOLDEN)
    groups, kw = ERRORS[case]
    expected = str(g["errors"][case])
    with pytest.raises(Exception) as info:
        sq.tl.var_by_distance(make_adata(AnnDataLite), groups_arg(groups), copy=True, **kw)
    assert type(info.value).__name__ == expected


def test_non_planar_coordinates_are_not_implemented(host_kernel):
    adata = make_adata(AnnDataLite)
    adata.obsm["spatial"] = np.concatenate([adata.obsm["spatial"], np.zeros((adata.n_obs, 1))], axis=1)
    with pytest.raises(NotImplementedError, match="2-D"):
        sq.tl.var_by_distance(adata, "a", cluster_key="cluster", copy=True)


def test_pool_is_one_query_range_per_slide(host_kernel):
    adata = make_adata(AnnDataLite)
    sq.tl.var_by_distance(adata, ["a", "b", "c"], cluster_key="cluster", library_key="library", copy=True)
    pool, tasks = host_kernel[0]
    # s0 has a, b and c, s1 has a and b: five tasks over two query ranges, the finite rows of each slide
    assert tasks.shape[0] == 5
    assert len({(t[2], t[3]) for t in tasks}) == 2
    lib = adata.obs["library"].to_numpy()
    finite = ~np.isnan(adata.obsm["spatial"]).any(axis=1)
    assert sorted(int(t[3] - t[2]) for t in tasks) == sorted([int((finite & (lib == "s0")).sum())] * 3 + [int((finite & (lib == "s1")).sum())] * 2)
    assert np.isfinite(pool).all()
