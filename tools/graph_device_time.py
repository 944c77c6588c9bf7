"""Host versus device coordinates for the spatial graph builders at 1M hex spots (SURVEY configs[1] geometry).

For every builder option: the median of 5 calls with numpy coordinates (GPU search, scipy post-processing on the host,
scipy CSR result) and with the same coordinates as a torch CUDA tensor (search and post-processing on the GPU, torch
sparse_csr result), the two alternated call by call; plus nhood_enrichment end to end on the device-built graph.  Every
device call ends in a synchronise (the export waits for the graph).  ``--json PATH`` also writes the numbers as JSON.

    python tools/graph_device_time.py [--reps 5] [--side 1000] [--json PATH]
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
from squidpy_b200.gr import GridBuilder, KNNBuilder  # noqa: E402
from tools import synth  # noqa: E402


def _gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--side", type=int, default=1000)
    ap.add_argument("--json", default=None, help="write the numbers to this JSON file")
    args = ap.parse_args()
    co = synth.hex_coords(args.side, args.side)
    n = co.shape[0]
    dev = torch.tensor(co, device="cuda")
    lib = pd.Categorical.from_codes(np.arange(n) % 4, categories=[f"l{i}" for i in range(4)])  # 4 interleaved libraries
    rows = {
        "KNNBuilder(6)": lambda c: KNNBuilder(6).build(c),
        "KNNBuilder(6, set_diag=True)": lambda c: KNNBuilder(6, set_diag=True).build(c),
        "KNNBuilder(6, set_diag=True, percentile=99)": lambda c: KNNBuilder(6, set_diag=True, percentile=99.0).build(c),
        "KNNBuilder(6, transform='spectral')": lambda c: KNNBuilder(6, transform="spectral").build(c),
        "KNNBuilder(6, transform='cosine')": lambda c: KNNBuilder(6, transform="cosine").build(c),
        "GridBuilder(6)": lambda c: GridBuilder(6).build(c),
        "GridBuilder(6, n_rings=3)": lambda c: GridBuilder(6, n_rings=3).build(c),
        "spatial_neighbors_knn(6, library_key) 4 libraries": lambda c: sq.gr.spatial_neighbors_knn(adatas[id(c)], n_neighs=6, library_key="lib",
                                                                                                  copy=True),
    }
    obs = pd.DataFrame({"lib": lib}, index=pd.RangeIndex(n).astype(str))  # built once: not part of the timed calls
    adatas = {id(c): sq.AnnDataLite(obs=obs, obsm={"spatial": c}, shape=(n, 0)) for c in (co, dev)}
    out = {"gpu": _gpu_info(), "n_obs": n, "reps": args.reps, "rows": {}}
    print(out["gpu"], f"n={n}", flush=True)
    for name, fn in rows.items():
        fn(co), fn(dev)  # warm-up of both paths
        torch.cuda.synchronize()
        t = {"host": [], "device": []}
        for _ in range(args.reps):
            for tag, c in (("host", co), ("device", dev)):
                t0 = time.perf_counter()
                fn(c)
                torch.cuda.synchronize()
                t[tag].append(time.perf_counter() - t0)
        med = {k: float(np.median(v)) * 1e3 for k, v in t.items()}
        out["rows"][name] = {"host_ms": med["host"], "device_ms": med["device"], "host_runs_ms": [x * 1e3 for x in t["host"]],
                             "device_runs_ms": [x * 1e3 for x in t["device"]]}
        print(f"{name:52s} host {med['host']:9.1f} ms   device {med['device']:8.1f} ms", flush=True)
    # coordinates -> graph -> statistics, all on the device
    labels = pd.Series(pd.Categorical.from_codes(np.random.default_rng(0).integers(0, 30, n), categories=[f"c{i}" for i in range(30)]))
    e2e = []
    for rep in range(args.reps + 1):
        ad = synth.make_adata(dev, None, labels)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sq.gr.spatial_neighbors_grid(ad, n_neighs=6)
        t1 = time.perf_counter()
        sq.gr.nhood_enrichment(ad, "cluster", n_perms=1000, seed=0, copy=True)
        t2 = time.perf_counter()
        if rep:  # the first is the warm-up
            e2e.append((t1 - t0, t2 - t1))
    g, s = np.median(np.array(e2e), axis=0) * 1e3
    out["pipeline"] = {"spatial_neighbors_grid_ms": float(g), "nhood_enrichment_1000_perms_ms": float(s)}
    print(f"device coords -> spatial_neighbors_grid {g:.1f} ms -> nhood_enrichment(n_perms=1000) {s:.1f} ms", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
