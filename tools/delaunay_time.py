"""GPU time of the Delaunay graph (host and device coordinates) beside scipy.spatial.Delaunay on the same inputs.

Times are wall clock around calls that end in a device synchronise, after one warm-up call per input; the median of three.
Prints the card name and power limit read in the same run, and the points finished by pass 1 and pass 2."""

from __future__ import annotations

import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scipy.spatial import Delaunay  # noqa: E402

from squidpy_b200.gr import DelaunayBuilder, delaunay_2d  # noqa: E402
from tools import synth  # noqa: E402


def _med(f, reps=3):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def main() -> None:
    import torch

    log = open(sys.argv[1], "a") if len(sys.argv) > 1 and sys.argv[1] != "-" else sys.stdout  # optional file, line by line

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", file=log, flush=True)
    rng = np.random.default_rng(0)
    k = np.stack(np.meshgrid(np.arange(1000), np.arange(1000)), -1).reshape(-1, 2).astype(np.float64)
    inputs = {
        "uniform 100k": rng.uniform(0, 1e4, (100_000, 2)),
        "uniform 1M": rng.uniform(0, 1e4, (1_000_000, 2)),
        "uniform 4M": rng.uniform(0, 1e4, (4_000_000, 2)),
        "thomas 1M": synth.thomas_points(1_000_000),
        "hex 1M": synth.hex_coords(1000, 1000),
        "square 1000x1000": k[rng.permutation(k.shape[0])],
    }
    only = [a for a in sys.argv[2:]]  # optional subset of the input names, e.g. "square 1000x1000"
    for name, xy in inputs.items():
        if only and name not in only:
            continue
        _, _, counts = delaunay_2d(xy, pass_counts=True)
        host = _med(lambda: delaunay_2d(xy))
        d = torch.from_numpy(xy).cuda()
        b = DelaunayBuilder()
        b.build(d)
        torch.cuda.synchronize()

        def dev():
            b.build(d)
            torch.cuda.synchronize()

        devt = _med(dev)
        t0 = time.perf_counter()
        Delaunay(xy).vertex_neighbor_vertices
        sci = time.perf_counter() - t0
        print(f"{name:18s} host-coords sqb_delaunay_2d {host * 1e3:9.1f} ms | device builder {devt * 1e3:9.1f} ms | scipy {sci * 1e3:9.1f} ms "
              f"| pass1 {counts[0]} pass2 {counts[1]}", file=log, flush=True)


if __name__ == "__main__":
    main()
