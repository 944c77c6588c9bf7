"""tl.var_by_distance on the GPU against the same call with scikit-learn's KDTree in place of the kernel, at 1 M cells over
20 000 x 20 000 in 4 slides, 12 clusters and 3 anchors, on four anchor geometries: a uniform cluster, a centred disc of radius
2000, a hollow annulus (r 8000-8150) and three thin lines.  The coherent geometries are where a grid search would visit
thousands of empty cells per query; a hierarchy should not care.

    python tools/var_by_distance_time.py [--n 1000000] [--reps 5] [--out results.json]

Every repetition runs the GPU call and the restatement alternately and asserts identical frames.  Reports medians after one
warm-up call per geometry, the kernel time of the GPU call (``ctx.profile``), its split between the device call and the
host assembly, and the card with its power limit.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

EXTENT = 20000.0
GEOMETRIES = ("uniform", "disc", "annulus", "lines")


def geometry(name: str, n: int, seed: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """n uniform points over EXTENT^2 and the boolean mask of the anchor cells of the named geometry."""
    rng = np.random.default_rng(seed)
    xy = rng.random((n, 2)) * EXTENT
    c = EXTENT / 2
    r = np.hypot(xy[:, 0] - c, xy[:, 1] - c)
    if name == "uniform":
        mask = rng.integers(0, 12, n) == 0
    elif name == "disc":
        mask = r <= 2000.0
    elif name == "annulus":
        mask = (r >= 8000.0) & (r <= 8150.0)
    elif name == "lines":  # three 80-wide "vessels": a horizontal, a vertical and a diagonal one
        mask = (np.abs(xy[:, 1] - 5000.0) <= 40.0) | (np.abs(xy[:, 0] - 12000.0) <= 40.0) | (np.abs(xy[:, 1] - xy[:, 0]) <= 56.0)
    elif name == "corner":
        mask = np.zeros(n, dtype=bool)
        mask[np.argsort(np.hypot(xy[:, 0], xy[:, 1]))[:500]] = True
    else:
        raise ValueError(name)
    return xy, mask


def make_adata(name: str, n: int, n_slides: int = 4, seed: int = 0):
    """A slide-labelled AnnDataLite: 12 random clusters c0..c11, the geometry's cells relabelled `anchor`."""
    from squidpy_b200 import AnnDataLite

    xy, mask = geometry(name, n, seed)
    rng = np.random.default_rng(seed + 1)
    codes = rng.integers(1, 12, n)
    codes[mask] = 0
    obs = pd.DataFrame({"cluster": pd.Categorical.from_codes(codes, categories=["anchor"] + [f"c{i}" for i in range(1, 12)]),
                        "library": pd.Categorical.from_codes(rng.integers(0, n_slides, n), categories=[f"s{i}" for i in range(n_slides)])},
                       index=pd.Index([f"cell{i}" for i in range(n)]))
    return AnnDataLite(obs=obs, obsm={"spatial": xy}, shape=(n, 0))


KW = dict(cluster_key="cluster", library_key="library", copy=True)
GROUPS = ["anchor", "c1", "c2"]


def _card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"nvidia_smi": r.stdout.strip()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    args = ap.parse_args()

    import squidpy_b200 as sq
    from squidpy_b200.tl import _var_by_distance as vbd
    from tests import nearest_ref

    ctx = sq.default_context(0)
    gpu_fn = vbd.nn_min_dist
    split = {"device": 0.0}

    def timed_gpu(*a, **k):
        t0 = time.perf_counter()
        out = gpu_fn(*a, **k)
        split["device"] += time.perf_counter() - t0
        return out

    def host_fn(points, tasks, metric, n_out, *, ctx=None):
        return nearest_ref.eval_tasks(points, tasks, metric, n_out)

    res = {"card": _card(), "n": args.n, "slides": 4, "anchors": GROUPS, "reps": args.reps, "geometries": {}}
    for name in GEOMETRIES:
        adata = make_adata(name, args.n)
        vbd.nn_min_dist = timed_gpu
        sq.tl.var_by_distance(adata, GROUPS, **KW)  # warm-up
        t_gpu, t_host, t_dev, t_kernel = [], [], [], []
        for _ in range(args.reps):
            vbd.nn_min_dist = timed_gpu
            split["device"] = 0.0
            ctx.profile(True)
            ctx.profile_reset()
            # profile mode synchronises every launch; the kernel time is read from this call, the wall times from the next
            sq.tl.var_by_distance(adata, GROUPS, **KW)
            t_kernel.append(ctx.profile_get("misc")[0])
            ctx.profile(False)
            split["device"] = 0.0
            t0 = time.perf_counter()
            got = sq.tl.var_by_distance(adata, GROUPS, **KW)
            t_gpu.append(time.perf_counter() - t0)
            t_dev.append(split["device"])
            vbd.nn_min_dist = host_fn
            t0 = time.perf_counter()
            exp = sq.tl.var_by_distance(adata, GROUPS, **KW)
            t_host.append(time.perf_counter() - t0)
            pd.testing.assert_frame_equal(got, exp, check_exact=True)
        vbd.nn_min_dist = gpu_fn
        n_anchor = int((adata.obs["cluster"] == "anchor").sum())
        row = {"anchor_cells": n_anchor, "gpu_call_s": float(np.median(t_gpu)), "sklearn_call_s": float(np.median(t_host)),
               "device_call_s": float(np.median(t_dev)), "host_assembly_s": float(np.median(t_gpu) - np.median(t_dev)),
               "kernel_ms": float(np.median(t_kernel)), "speedup": float(np.median(t_host) / np.median(t_gpu))}
        res["geometries"][name] = row
        print(name, json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res["card"]))


if __name__ == "__main__":
    main()
