"""interaction_matrix(weights=True) at 1M spots (a 1000 x 1000 hexagonal lattice, 6 M stored entries) on the GPU, from a host
graph (scipy CSR) and from a device graph (torch sparse_csr, int64 indices).

Weights: the lattice's binary connectivities (float32 ones: every partial sum is an exact integer, the atomics path) and random
float32 weights drawn as float64 and rounded (not on a common 2^-24 grid: the ordered path) at C = 2, 20, 300 and 4096 random
clusters.  Per leg: the whole call (host clock around a call whose result is copied to the host, so it ends in a device
synchronise), one warm-up, then ``--reps`` calls with the legs alternated, median.

``--compare TREE`` times another checkout of the package (built in place) against this one: the two run in alternating
worker processes, ``--rounds`` each, and each leg reports the median over all of a tree's calls.  Prints the card and its
power limit; ``--out FILE`` also writes the results as JSON.

    python tools/interaction_time.py [--reps 5] [--compare TREE --rounds 3] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLUSTERS = (2, 20, 300, 4096)


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() or "unknown"


def worker(root: str, reps: int) -> dict:
    """Times every leg with the package of ``root``; returns {leg: [seconds, ...]}."""
    sys.path.insert(0, root)
    import numpy as np
    import pandas as pd
    import scipy.sparse as sp
    import torch

    import squidpy_b200 as sq
    from squidpy_b200 import AnnDataLite
    from tools import synth

    g = synth.hex_graph(1000, 1000)
    n = g.shape[0]
    rng = np.random.default_rng(0)
    graphs = {"binary": g, "f32": sp.csr_matrix((rng.random(g.nnz).astype(np.float32), g.indices, g.indptr), shape=g.shape)}
    legs = {}
    for wname, h in graphs.items():
        dev = torch.sparse_csr_tensor(torch.from_numpy(h.indptr.astype(np.int64)), torch.from_numpy(h.indices.astype(np.int64)),
                                      torch.from_numpy(h.data), size=h.shape).cuda()
        for k in (20,) if wname == "binary" else CLUSTERS:
            cat = pd.Categorical.from_codes(rng.integers(0, k, n), categories=[f"c{i}" for i in range(k)])
            obs = pd.DataFrame({"cl": cat})
            for where, m in (("host", h), ("device", dev)):
                legs[f"{where} {wname} C={k}"] = AnnDataLite(obs=obs, obsp={"spatial_connectivities": m}, shape=(n, 1))
    sq.default_context(0)
    times = {name: [] for name in legs}
    for rep in range(reps + 1):
        for name, ad in legs.items():
            t0 = time.perf_counter()
            sq.gr.interaction_matrix(ad, "cl", weights=True, copy=True)
            if rep:  # the first round warms every leg up
                times[name].append(time.perf_counter() - t0)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--compare", default=None, help="another checkout of the package, timed against this one")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        print(json.dumps(worker(a.worker, a.reps)))
        return
    info = card()
    print("card, power limit:", info, flush=True)
    trees = {"this": HERE} if a.compare is None else {"other": os.path.abspath(a.compare), "this": HERE}
    times: dict = {t: {} for t in trees}
    for _ in range(a.rounds if a.compare else 1):
        for t, root in trees.items():
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", root, "--reps", str(a.reps)], capture_output=True,
                               text=True, check=True)
            for leg, ts in json.loads(r.stdout.strip().splitlines()[-1]).items():
                times[t].setdefault(leg, []).extend(ts)
    import numpy as np

    med = {t: {leg: float(np.median(ts)) for leg, ts in legs.items()} for t, legs in times.items()}
    for leg in med["this"]:
        line = f"{leg:24s} this {med['this'][leg] * 1e3:9.2f} ms"
        if "other" in med:
            line += f"   other {med['other'][leg] * 1e3:9.2f} ms   this / other {med['this'][leg] / med['other'][leg]:.2f}"
        print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "median_s": med, "calls": times}, f, indent=1)


if __name__ == "__main__":
    main()
