"""Generates tests/golden/ripley_l_metrics.npz: the UNMODIFIED reference ``ripley`` (``/root/reference/src/squidpy``, through
the stub-import loader ``oracle/_refload.py``) in mode L for all nine metric names ``KDTree`` takes.  Only runnable where the
reference tree exists; the output is committed.

    python tests/golden/make_golden_ripley_l_metrics.py

Fixture: the integer lattice of ``make_golden_ripley_fg`` (a 10 x 10 block, an 8 x 6 block, clusters of 5 and 6 points)
plus a cluster of one point.  Per metric: the default ``max_dist``; ``max_dist=12`` with 13 steps, so every edge is an
integer and lattice pairs lie exactly on it in all three distances; ``max_dist=0``, which repeats one edge five times.
"""

from __future__ import annotations

import os
import sys

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import _refload  # noqa: E402
from squidpy_b200._adata import AnnDataLite  # noqa: E402
from tests.golden import make_golden_ripley_fg  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

METRICS = ["euclidean", "l2", "minkowski", "p", "manhattan", "cityblock", "l1", "chebyshev", "infinity"]
# (n_steps, max_dist, n_observations)
SHAPES = [(50, None, 50), (13, 12.0, 50), (5, 0.0, 30)]
CASES = [(metric, *shape) for metric in METRICS for shape in SHAPES]
N_SIM, SEED = 10, 7
CATEGORIES = ["a", "b", "c", "d", "e"]


def fixture():
    xy, codes = make_golden_ripley_fg.fixture()
    return np.concatenate([xy, [[15.0, 20.0]]]), np.concatenate([codes, [4]])  # "e": a cluster of one point


def make_adata(xy, codes):
    obs = pd.DataFrame({"cluster": pd.Categorical.from_codes(codes, categories=CATEGORIES)}, index=[str(i) for i in range(len(codes))])
    return AnnDataLite(X=np.zeros((len(codes), 1)), obs=obs, var=pd.DataFrame(index=["g0"]), obsm={"spatial": xy.copy()})


def main():
    import sklearn

    rp = _refload.load()["rp"]
    xy, codes = fixture()
    out = {"meta": np.array(f"numpy {np.__version__}; sklearn {sklearn.__version__}; reference squidpy ripley mode L, "
                            f"n_simulations={N_SIM}, seed={SEED}"), "xy": xy, "codes": codes}
    for i, (metric, n_steps, max_dist, n_obs) in enumerate(CASES):
        res = rp.ripley(make_adata(xy, codes), "cluster", mode="L", metric=metric, n_simulations=N_SIM, n_observations=n_obs,
                        max_dist=max_dist, n_steps=n_steps, seed=SEED, copy=True)
        out[f"c{i}_stat"] = res["L_stat"]["stats"].to_numpy()
        out[f"c{i}_sims"] = res["sims_stat"]["stats"].to_numpy()
        out[f"c{i}_bins"] = res["bins"]
        out[f"c{i}_pvalues"] = res["pvalues"]
    np.savez_compressed(os.path.join(OUT, "ripley_l_metrics.npz"), **out)
    print("wrote ripley_l_metrics.npz", len(CASES), "cases")


if __name__ == "__main__":
    main()
