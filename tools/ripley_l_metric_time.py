"""ripley(mode="L") per metric class at configs[4] (300 000 Thomas points, 12 Dirichlet clusters, 100 simulations of 1000
points, 50 radii): the pair-count kernel (CUDA events, ctx.profile), the whole ``ripley()`` call, and the same counts from
scikit-learn's ``KDTree(g, metric=m).two_point_correlation(g, support, dualtree=True)``.  The GPU legs of the three metrics
are alternated, median of ``--reps`` calls after one warm-up of each.  scikit-learn runs every group (the 12 clusters and the
100 simulations) on a pool of ``--jobs`` processes, ``--sklearn-reps`` times per metric; its counts must equal the GPU's.
Prints the card and its power limit; ``--out FILE`` also writes the results as JSON.

    python tools/ripley_l_metric_time.py [--reps 3] [--sklearn-reps 1] [--jobs 0] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import multiprocessing
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import squidpy_b200 as sq  # noqa: E402
from squidpy_b200.gr import _ripley  # noqa: E402
from tools import synth  # noqa: E402

METRICS = ("euclidean", "manhattan", "chebyshev")


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() or "unknown"


def _tpc(args):
    from sklearn.neighbors import KDTree

    g, support, metric = args
    return KDTree(g, metric=metric).two_point_correlation(g, support, dualtree=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sklearn-reps", type=int, default=1)
    ap.add_argument("--jobs", type=int, default=0, help="scikit-learn worker processes (0: one per core)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    ctx = sq.default_context(0)
    info = card()
    print("card, power limit:", info)
    n = 300_000
    pts = synth.thomas_points(n, seed=5)
    ad = synth.make_adata(pts, None, synth.dirichlet_labels(n, 12, seed=5))
    kw = dict(mode="L", n_steps=50, n_simulations=100, n_observations=1000, seed=0, copy=True)

    # the groups and support one ripley() call hands to pair_counts, for the scikit-learn leg
    captured = {}
    real = _ripley.pair_counts

    def capture(groups, support, **k):
        captured["groups"], captured["support"] = [np.array(g) for g in groups], np.array(support)
        out = real(groups, support, **k)
        captured[k["metric"]] = out
        return out

    _ripley.pair_counts = capture
    try:
        for m in METRICS:
            sq.gr.ripley(ad, "cluster", metric=m, **kw)  # warm-up, and the counts of each metric
    finally:
        _ripley.pair_counts = real

    call, kern = {m: [] for m in METRICS}, {m: [] for m in METRICS}
    for _ in range(a.reps):
        for m in METRICS:
            ctx.profile(True)
            ctx.profile_reset()
            t0 = time.perf_counter()
            sq.gr.ripley(ad, "cluster", metric=m, **kw)
            call[m].append(time.perf_counter() - t0)
            kern[m].append(ctx.profile_get("pairs")[0])
            ctx.profile(False)

    groups, support = captured["groups"], captured["support"]
    jobs = a.jobs or len(os.sched_getaffinity(0))
    order = sorted(range(len(groups)), key=lambda i: -len(groups[i]))  # largest groups first: they bound the wall time
    skl = {m: [] for m in METRICS}
    with ProcessPoolExecutor(jobs, mp_context=multiprocessing.get_context("spawn")) as pool:  # no fork of the CUDA process
        for _ in range(a.sklearn_reps):
            for m in METRICS:
                t0 = time.perf_counter()
                res = list(pool.map(_tpc, [(groups[i], support, m) for i in order]))
                skl[m].append(time.perf_counter() - t0)
                counts = np.empty((len(groups), support.size), np.int64)
                counts[order] = np.stack(res)
                assert np.array_equal(counts, captured[_ripley.metric_code(m)]), f"{m}: GPU counts differ from scikit-learn"

    pairs = float(sum(len(g) ** 2 for g in groups))
    rows = {}
    for m in METRICS:
        rows[m] = {"kernel_ms_median": float(np.median(kern[m])), "kernel_ms": kern[m], "ripley_s_median": float(np.median(call[m])),
                   "ripley_s": call[m], "sklearn_s_median": float(np.median(skl[m])), "sklearn_s": skl[m],
                   "kernel_pairs_per_s": pairs / (np.median(kern[m]) / 1e3)}
        print(f"{m:9s}: pair-count kernel median {rows[m]['kernel_ms_median']:.2f} ms ({rows[m]['kernel_pairs_per_s'] / 1e9:.1f} G pairs/s), "
              f"ripley() median {rows[m]['ripley_s_median']:.3f} s, scikit-learn two_point_correlation {rows[m]['sklearn_s_median']:.1f} s "
              f"on {jobs} processes; counts identical")
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card_power_limit": info, "ordered_pairs": pairs, "groups": len(groups), "radii": int(support.size), "reps": a.reps,
                       "sklearn_reps": a.sklearn_reps, "sklearn_jobs": jobs, "metrics": rows}, f, indent=1)


if __name__ == "__main__":
    main()
