"""centrality_scores at 1M spots (a 1000 x 1000 hexagonal lattice) on the GPU, against networkx at the largest lattice it
finishes within ``--nx-budget`` seconds.

GPU legs: 20 and 150 clusters, each with random labels (every node a few hops from every cluster: a shallow BFS) and with
stripes of columns (spatially coherent clusters: a BFS as deep as the lattice is wide).  Per leg: the whole
``centrality_scores`` call and ``centrality_counts`` alone (host clock around calls that end in a device synchronise),
median of ``--reps`` after one warm-up, and the BFS level count.  networkx leg: ``group_degree_centrality``,
``group_closeness_centrality`` and ``average_clustering`` for every cluster on lattices of growing size, 20 random
clusters; its degree and closeness must equal the GPU's, its clustering means differ from numpy's pairwise mean in the last
bits at most.  The reference's own rustworkx path is not measured (rustworkx is not
installed).  Prints the card and its power limit; ``--out FILE`` also writes the results as JSON.

    python tools/centrality_time.py [--reps 3] [--nx-budget 120] [--out FILE]
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import squidpy_b200 as sq  # noqa: E402
from squidpy_b200.gr import centrality_counts  # noqa: E402
from tools import synth  # noqa: E402


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() or "unknown"


def labels(side: int, n_cls: int, stripes: bool) -> np.ndarray:
    n = side * side
    if stripes:
        return (np.arange(n) % side) * n_cls // side
    return np.random.default_rng(n_cls).integers(0, n_cls, n)


def adata(g, codes, n_cls):
    cats = pd.Categorical.from_codes(codes, categories=[f"c{i}" for i in range(n_cls)])
    return synth.make_adata(synth.hex_coords(int(np.sqrt(g.shape[0])), int(np.sqrt(g.shape[0]))), g, pd.Series(cats))


def gpu_leg(g, n_cls, stripes, reps):
    codes = labels(1000, n_cls, stripes)
    ad = adata(g, codes, n_cls)
    sq.gr.centrality_scores(ad, "cluster", copy=True)  # warm-up
    t_call, t_counts = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        sq.gr.centrality_scores(ad, "cluster", copy=True)
        t_call.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        res = centrality_counts(g, codes.astype(np.int32), n_cls, 7)
        t_counts.append(time.perf_counter() - t0)
    return {"clusters": n_cls, "labels": "stripes" if stripes else "random", "call_s": float(np.median(t_call)),
            "counts_s": float(np.median(t_counts)), "bfs_levels": res.levels}


def nx_leg(side, n_cls=20):
    import networkx as nx

    g = synth.hex_graph(side, side)
    codes = labels(side, n_cls, False)
    t0 = time.perf_counter()
    G = nx.Graph(g)
    rows = []
    for k in range(n_cls):
        idx = np.flatnonzero(codes == k).tolist()
        rows.append((nx.group_degree_centrality(G, idx), nx.average_clustering(G, idx), nx.group_closeness_centrality(G, idx)))
    t = time.perf_counter() - t0
    got = sq.gr.centrality_scores(adata(g, codes, n_cls), "cluster", copy=True).to_numpy()
    exp = np.array(rows)
    # networkx averages the clustering coefficients with Python's sequential sum, the reference with numpy's pairwise mean
    return {"spots": side * side, "clusters": n_cls, "networkx_s": t,
            "degree_closeness_equal": bool(np.array_equal(got[:, [0, 2]], exp[:, [0, 2]])),
            "clustering_max_abs_diff": float(np.abs(got[:, 1] - exp[:, 1]).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--nx-budget", type=float, default=120.0, help="stop growing the networkx lattice after a run this long")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sq.default_context(0)
    info = card()
    print("card, power limit:", info)
    g = synth.hex_graph(1000, 1000)
    out = {"card": info, "gpu": [], "networkx": []}
    for n_cls in (20, 150):
        for stripes in (False, True):
            r = gpu_leg(g, n_cls, stripes, a.reps)
            out["gpu"].append(r)
            print(f"GPU 1M spots, {n_cls} clusters, {r['labels']:7s}: centrality_scores {r['call_s'] * 1e3:8.1f} ms, "
                  f"counts {r['counts_s'] * 1e3:8.1f} ms, {r['bfs_levels']} BFS levels", flush=True)
    for side in (50, 100, 200, 400):
        r = nx_leg(side)
        out["networkx"].append(r)
        print(f"networkx {r['spots']} spots, 20 clusters: {r['networkx_s']:.1f} s; degree and closeness equal to the GPU's: "
              f"{r['degree_closeness_equal']}, clustering within {r['clustering_max_abs_diff']:.1e}", flush=True)
        if r["networkx_s"] > a.nx_budget:
            break
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
