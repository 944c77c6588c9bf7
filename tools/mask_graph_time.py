"""Wall-clock times of ``mask_graph`` on 1M-observation graphs: a hex lattice and uniform points, their kNN(6) and Delaunay graphs,
from the host (scipy CSR, numpy coordinates) and from GPU memory (torch sparse_csr, device coordinates), masked by a star-shaped
polygon of 10^4 shell vertices with four holes.  Each time is the median of three calls ending in a device synchronise, after a
warm-up call; the GPU's name and power limit are read in the same run.  Writes a JSON line to stdout and to ``--out``.

    python tools/mask_graph_time.py --out results/mask_graph_time.json
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200._adata import AnnDataLite  # noqa: E402


def gpu_info() -> str:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def hex_points(n: int) -> np.ndarray:
    side = int(np.sqrt(n))
    i, j = np.meshgrid(np.arange(side), np.arange(side))
    return np.c_[(i + 0.5 * (j % 2)).ravel(), (j * np.sqrt(3) / 2).ravel()].astype(np.float64) * (1000.0 / side)


class Geo:
    def __init__(self, kind, coordinates):
        self.__geo_interface__ = {"type": kind, "coordinates": coordinates}


def polygon(rng, k: int, c: float, r: float) -> Geo:
    def ring(m, cx, cy, rr):
        ang = np.sort(rng.uniform(0, 2 * np.pi, m))
        rad = rr * rng.uniform(0.85, 1.0, m)
        return tuple(map(tuple, np.c_[cx + rad * np.cos(ang), cy + rad * np.sin(ang)]))

    holes = [ring(k // 20, c + 0.4 * r * np.cos(a), c + 0.4 * r * np.sin(a), 0.1 * r) for a in np.arange(4) * np.pi / 2]
    return Geo("Polygon", (ring(k, c, c, r), *holes))


def median_time(fn, sync, reps: int = 3) -> float:
    fn()
    sync()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        sync()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--vertices", type=int, default=10_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    sync = torch.cuda.synchronize
    rng = np.random.default_rng(0)
    geom = polygon(rng, args.vertices, 500.0, 450.0)
    rows = []
    for layout, pts in (("hex", hex_points(args.n)), ("uniform", rng.uniform(0, 1000, (args.n, 2)))):
        for graph in ("knn6", "delaunay"):
            build = (lambda a: sq.gr.spatial_neighbors_knn(a, n_neighs=6)) if graph == "knn6" else sq.gr.spatial_neighbors_delaunay
            h = AnnDataLite(shape=(len(pts), 0))
            h.obsm["spatial"] = pts
            build(h)
            d = AnnDataLite(shape=(len(pts), 0))
            d.obsm["spatial"] = torch.as_tensor(pts, device="cuda")
            build(d)
            nnz = h.obsp["spatial_connectivities"].nnz
            kept = sq.gr.mask_graph(h, None, geom, copy=True)[0].nnz
            t_host = median_time(lambda: sq.gr.mask_graph(h, None, geom, copy=True), sync)
            t_dev = median_time(lambda: sq.gr.mask_graph(d, None, geom, copy=True), sync)
            rows.append({"points": layout, "graph": graph, "n": len(pts), "edges": nnz, "kept": kept, "host_graph_s": t_host, "device_graph_s": t_dev})
            print(json.dumps(rows[-1]), flush=True)
    res = {"gpu": gpu_info(), "polygon_shell_vertices": args.vertices, "polygon_hole_vertices": 4 * (args.vertices // 20), "rows": rows}
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
