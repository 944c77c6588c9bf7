"""Generates tests/golden/ripley_fg.npz: the UNMODIFIED reference ``ripley`` (``/root/reference/src/squidpy``, through the
stub-import loader ``oracle/_refload.py``) in modes F and G on a fixture that reaches every edge case of the device
search and binning at once.  Only runnable where the reference tree exists; the output is committed.

    python tests/golden/make_golden_ripley_fg.py

Fixture: an integer lattice of four spatially segregated clusters -- a 10 x 10 block, an 8 x 6 block on the far side, a
cluster of 5 points (n_neigh=2: scikit-learn's brute force) and one of 6 (its kd_tree).  Integer support edges make
lattice distances fall exactly on edges; small ``max_dist`` values drop distances above the last edge; ``max_dist=0``
repeats every edge; ``n_observations=4`` leaves every simulation to brute force; metrics euclidean and minkowski.
"""

from __future__ import annotations

import os
import sys
import warnings

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import _refload  # noqa: E402
from squidpy_b200._adata import AnnDataLite  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

# (mode, metric, n_steps, max_dist, n_observations)
CASES = [
    ("G", "euclidean", 50, None, 50),
    ("F", "euclidean", 50, None, 50),
    ("G", "minkowski", 13, 12.0, 50),
    ("F", "minkowski", 13, 12.0, 50),
    ("G", "euclidean", 2, 3.0, 50),
    ("F", "euclidean", 2, 3.0, 50),
    ("G", "minkowski", 50, 20.0, 4),
    ("F", "euclidean", 13, 12.0, 4),
    ("G", "euclidean", 5, 0.0, 50),
]
N_SIM, SEED = 10, 11


def fixture():
    gx, gy = np.meshgrid(np.arange(10), np.arange(10))
    a = np.stack([gx.ravel(), gy.ravel()], 1)
    gx, gy = np.meshgrid(np.arange(40, 48), np.arange(0, 6))
    b = np.stack([gx.ravel(), gy.ravel()], 1)
    c = np.stack([np.arange(20, 25), np.full(5, 30)], 1)
    d = np.stack([np.arange(30, 36), np.full(6, 40)], 1)
    xy = np.concatenate([a, b, c, d]).astype(np.float64)
    codes = np.repeat(np.arange(4), [len(a), len(b), len(c), len(d)])
    perm = np.random.default_rng(0).permutation(len(codes))  # clusters interleaved in observation order
    return xy[perm], codes[perm]


def make_adata(xy, codes):
    obs = pd.DataFrame({"cluster": pd.Categorical.from_codes(codes, categories=["a", "b", "c", "d"])}, index=[str(i) for i in range(len(codes))])
    return AnnDataLite(X=np.zeros((len(codes), 1)), obs=obs, var=pd.DataFrame(index=["g0"]), obsm={"spatial": xy.copy()})


def main():
    import sklearn

    rp = _refload.load()["rp"]
    xy, codes = fixture()
    out = {"meta": np.array(f"numpy {np.__version__}; sklearn {sklearn.__version__}; reference squidpy ripley, n_neigh=2, "
                            f"n_simulations={N_SIM}, seed={SEED}"), "xy": xy, "codes": codes}
    for i, (mode, metric, n_steps, max_dist, n_obs) in enumerate(CASES):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")  # max_dist=0: every count is 0, the fractions are NaN
            res = rp.ripley(make_adata(xy, codes), "cluster", mode=mode, metric=metric, n_neigh=2, n_simulations=N_SIM,
                            n_observations=n_obs, max_dist=max_dist, n_steps=n_steps, seed=SEED, copy=True)
        out[f"c{i}_stat"] = res[f"{mode}_stat"]["stats"].to_numpy()
        out[f"c{i}_sims"] = res["sims_stat"]["stats"].to_numpy()
        out[f"c{i}_bins"] = res["bins"]
        out[f"c{i}_pvalues"] = res["pvalues"]
    np.savez_compressed(os.path.join(OUT, "ripley_fg.npz"), **out)
    print("wrote ripley_fg.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
