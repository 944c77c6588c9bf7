"""GPU parity tests of sepal (SURVEY.md 8f-4) against scores produced by the UNMODIFIED reference (tests/golden/sepal.npz).
The score is dt x (iteration at which the entropy change drops to 1e-8); the reference runs under numba fastmath, so an
iteration count may differ by a step or two where the entropy change grazes the threshold — most genes must agree exactly."""

from __future__ import annotations

import os

import numpy as np
import pandas as pd
import pytest

import squidpy_b200 as sq
from squidpy_b200.gr import sepal_scores
from squidpy_b200.gr._sepal import _compute_idxs
from tests.golden.make_golden_sepal import make_case

pytestmark = pytest.mark.gpu
GOLD = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "sepal.npz"), allow_pickle=False))
DT = 0.001


@pytest.mark.parametrize("name", ["hex", "square"])
def test_scores_match_reference_golden(name):
    g, co, k, vals = make_case(name)
    sat, sat_idx, unsat, unsat_idx = _compute_idxs(g, co, k)
    for key, arr in (("sat", sat), ("sat_idx", sat_idx), ("unsat", unsat), ("unsat_idx", unsat_idx)):
        np.testing.assert_array_equal(arr, GOLD[f"{name}_{key}"])  # host bookkeeping == the reference's _compute_idxs
    got = sepal_scores(vals, sat, sat_idx, unsat, unsat_idx, max_neighs=k)
    exp = GOLD[f"{name}_score"]
    assert np.array_equal(np.isnan(got), np.isnan(exp))
    ok = ~np.isnan(exp)
    d_iter = np.abs(got[ok] - exp[ok]) / DT
    assert (d_iter <= 2.5).all(), d_iter
    assert (d_iter < 0.5).mean() >= 0.8
    short = sepal_scores(vals, sat, sat_idx, unsat, unsat_idx, max_neighs=k, n_iter=300)
    np.testing.assert_array_equal(np.isnan(short), np.isnan(GOLD[f"{name}_score_300"]))  # not converged in 300 iterations -> NaN
    import scipy.sparse as sp

    np.testing.assert_array_equal(sepal_scores(sp.csr_matrix(vals), sat, sat_idx, unsat, unsat_idx, max_neighs=k), got)


def test_api_and_errors():
    g, co, k, vals = make_case("hex")
    genes = [f"g{i}" for i in range(vals.shape[1])]
    ad = sq.AnnDataLite(X=vals, obs=pd.DataFrame(index=[str(i) for i in range(vals.shape[0])]), var=pd.DataFrame(index=genes),
                        obsm={"spatial": co}, obsp={"spatial_connectivities": g})
    df = sq.gr.sepal(ad, max_neighs=6, copy=True)
    assert list(df.columns) == ["sepal_score"] and df.shape == (len(genes), 1)
    assert (np.diff(df["sepal_score"].dropna().to_numpy()) <= 0).all()  # sorted descending
    sq.gr.sepal(ad, max_neighs=6, genes=["g3", "g1"])
    assert set(ad.uns["sepal_score"].index) == {"g3", "g1"}
    with pytest.raises(ValueError, match="max_neighs"):
        sq.gr.sepal(ad, max_neighs=5)
    with pytest.raises(ValueError, match="found node with"):
        sq.gr.sepal(ad, max_neighs=4)


def test_large_lattice_uses_global_scratch():
    """160 x 160 spots: 2 x 8 B x 25 600 no longer fits shared memory -> per-CTA global scratch; checked against the numpy
    restatement of the diffusion loop (oracle.ref.sepal_score, plain float64): the same stopping iteration, exactly, on every
    gene whose decisions are well conditioned (tests/test_gpu_sepal_exact.py)."""
    from oracle import ref
    from tests.device_attrs import smem_optin
    from tests.test_gpu_sepal_exact import assert_exact, diffusion_trajectory, uses_global_scratch
    from tools import synth

    g, co = synth.hex_graph(160, 160), synth.hex_coords(160, 160)
    assert uses_global_scratch(g.shape[0], smem_optin())
    rng = np.random.default_rng(0)
    vals = np.stack([rng.random(len(co)) * (1 + q) + (q == 2) * rng.poisson(0.2, len(co)) for q in range(3)], axis=1)
    sat, sat_idx, unsat, unsat_idx = _compute_idxs(g, co, 6)
    a = sepal_scores(vals, sat, sat_idx, unsat, unsat_idx, max_neighs=6, n_iter=1500)
    np.testing.assert_array_equal(a, sepal_scores(vals, sat, sat_idx, unsat, unsat_idx, max_neighs=6, n_iter=1500))
    exp = np.array([ref.sepal_score(vals[:, q], True, 1500, sat, sat_idx, unsat, unsat_idx) for q in range(3)])
    assert np.isfinite(exp).any()
    traj = diffusion_trajectory(vals, True, 1500, sat, sat_idx, unsat, unsat_idx)
    np.testing.assert_array_equal(traj.scores(DT), exp)
    assert_exact(a, traj, DT, both_outcomes=False, min_conditioned=1.0)
