"""ripley(mode="F" / "G") at configs[4] (300 000 Thomas points, 12 clusters, 100 simulations of 1000 points): the GPU
call against the host path (scikit-learn for every set), calls alternated, median of the timed calls after one warm-up
of each; the search kernels' time from ctx.profile; both labellings (random Dirichlet labels and clusters as spatial
blocks).  Asserts that both paths return identical results, and prints the card and its power limit.

    python tools/ripley_fg_time.py [--reps 3] [--modes G,F] [--labels random,region]
"""

from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import pandas as pd

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import squidpy_b200 as sq  # noqa: E402
from squidpy_b200.gr import _ripley  # noqa: E402
from tools import synth  # noqa: E402


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() or "unknown"


def region_labels(pts: np.ndarray, n: int) -> pd.Series:
    x = pts[:, 0]
    codes = np.minimum(((x - x.min()) / (np.ptp(x) + 1e-9) * n).astype(int), n - 1)
    return pd.Series(pd.Categorical.from_codes(codes, categories=[f"r{i:02d}" for i in range(n)]))


def run(ad, mode: str, host: bool):
    kd = _ripley._kd_tree_euclidean
    if host:
        _ripley._kd_tree_euclidean = lambda metric, n_neigh, n_fit: False
    try:
        t0 = time.perf_counter()
        res = sq.gr.ripley(ad, "cluster", mode=mode, n_simulations=100, n_observations=1000, seed=0, copy=True)
        return time.perf_counter() - t0, res
    finally:
        _ripley._kd_tree_euclidean = kd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--modes", default="G,F")
    ap.add_argument("--labels", default="random,region")
    a = ap.parse_args()
    ctx = sq.default_context(0)
    print("card, power limit:", card())
    pts = synth.thomas_points(300_000, seed=5)
    labellings = {"random": synth.dirichlet_labels(300_000, 12, seed=5), "region": region_labels(pts, 12)}
    labellings = {k: labellings[k] for k in a.labels.split(",")}
    warnings.simplefilter("ignore")
    for mode in a.modes.split(","):
        for name, lab in labellings.items():
            ad = synth.make_adata(pts, None, lab)
            run(ad, mode, False), run(ad, mode, True)  # warm-up
            tg, th, kern = [], [], []
            for _ in range(a.reps):
                ctx.profile(True)
                ctx.profile_reset()
                dt, dev = run(ad, mode, False)
                kern.append(ctx.profile_get("misc")[0])
                ctx.profile(False)
                tg.append(dt)
                dt, host = run(ad, mode, True)
                th.append(dt)
                assert dev[f"{mode}_stat"].equals(host[f"{mode}_stat"]) and dev["sims_stat"].equals(host["sims_stat"])
                assert np.array_equal(dev["pvalues"], host["pvalues"])
            print(f"ripley {mode} {name:6s}: GPU call median {np.median(tg):.3f} s, host path median {np.median(th):.3f} s, "
                  f"speed-up {np.median(th) / np.median(tg):.1f}x, device kernels (profiled) median {np.median(kern):.2f} ms; outputs identical")


if __name__ == "__main__":
    main()
