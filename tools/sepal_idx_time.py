"""Wall-clock times of sepal's saturation tables: ``sepal_idxs`` (built on the GPU, ``sqb_sepal_idxs``) against the host
restatement ``_compute_idxs`` (the copy path), and the whole ``sepal(copy=True)`` call, on square 4-neighbour lattices with a
random fraction of the spots removed (what a tissue mask does to Visium HD / Stereo-seq bins) and on a full hex lattice.

The GPU tables are timed from a host graph (scipy CSR, numpy coordinates) and from GPU memory (torch ``sparse_csr``, CUDA
coordinates); ``_compute_idxs`` on the host CSR (it has no zeros to eliminate).  ``sepal`` is timed with the tables built on the
GPU from either graph, and from the host graph with the tables from ``_compute_idxs`` (how ``sepal`` built them before).  Every
time is the median of ``--reps`` alternated calls ending in a device synchronise, after a warm-up call; every GPU table is
checked equal to ``_compute_idxs`` and every ``sepal`` frame to the others.  The ``sepal`` call scores 4 genes with
``n_iter=100`` so that the tables weigh in it.  The GPU's name and power limit are read in the same run.  Writes a JSON line
to stdout and to ``--out``.

    python tools/sepal_idx_time.py --out results/sepal_idx_time.json
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools import synth  # noqa: E402

CASES = (("square", 300, 0.02), ("square", 600, 0.02), ("square", 1000, 0.01), ("hex", 300, 0.0))


def gpu_info() -> str:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def lattice(kind: str, side: int, drop: float, seed: int = 0) -> tuple[sp.csr_matrix, np.ndarray, int]:
    """``(graph, coordinates, max_neighs)``: a side x side square 4-neighbour or hex 6-neighbour lattice (CSR float32 ones,
    int32 sorted indices) without a random fraction ``drop`` of its spots."""
    if kind == "hex":
        g, co, k = synth.hex_graph(side, side), synth.hex_coords(side, side), 6
    else:
        idx = np.arange(side * side).reshape(side, side)
        src = np.r_[idx[:, :-1].ravel(), idx[:, 1:].ravel(), idx[:-1, :].ravel(), idx[1:, :].ravel()]
        dst = np.r_[idx[:, 1:].ravel(), idx[:, :-1].ravel(), idx[1:, :].ravel(), idx[:-1, :].ravel()]
        g = sp.csr_matrix((np.ones(src.size, np.float32), (src, dst)), shape=(side * side,) * 2)
        co = np.stack(np.meshgrid(np.arange(side, dtype=float), np.arange(side, dtype=float)), -1).reshape(-1, 2)
        k = 4
    keep = np.flatnonzero(np.random.default_rng(seed).random(side * side) >= drop)
    g = g[keep][:, keep].tocsr()
    g.sort_indices()
    g.indptr, g.indices = g.indptr.astype(np.int32), g.indices.astype(np.int32)
    return g, co[keep], k


def median_time(fns: dict, sync, reps: int) -> dict:
    """Median wall time of each callable, the calls alternated round by round after one warm-up round."""
    for fn in fns.values():
        fn()
    sync()
    ts = {name: [] for name in fns}
    for _ in range(reps):
        for name, fn in fns.items():
            t0 = time.perf_counter()
            fn()
            sync()
            ts[name].append(time.perf_counter() - t0)
    return {name: float(np.median(v)) for name, v in ts.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import pandas as pd
    import torch

    import squidpy_b200 as sq
    from squidpy_b200._adata import AnnDataLite
    from squidpy_b200.gr import _sepal
    from squidpy_b200.gr._sepal import _compute_idxs, _host_idxs, sepal_idxs

    def sepal_host_tables(ad, k):
        """The whole call with the tables from ``_compute_idxs`` on host copies, as sepal built them before sqb_sepal_idxs."""
        _sepal.sepal_idxs = lambda conn, spatial, max_neighs, device=None: _host_idxs(conn, spatial, max_neighs)
        try:
            return sq.gr.sepal(ad, max_neighs=k, n_iter=100, copy=True)
        finally:
            _sepal.sepal_idxs = sepal_idxs

    sync = torch.cuda.synchronize
    rows = []
    for kind, side, drop in CASES:
        g, co, k = lattice(kind, side, drop)
        n = g.shape[0]
        g_dev = torch.sparse_csr_tensor(torch.as_tensor(g.indptr), torch.as_tensor(g.indices), torch.as_tensor(g.data), size=g.shape).cuda()
        co_dev = torch.as_tensor(co).cuda()
        ref = _compute_idxs(g, co, k)
        for got in (sepal_idxs(g, co, k), sepal_idxs(g_dev, co_dev, k)):
            assert all(np.array_equal(a, b) for a, b in zip(got, ref)), f"{kind} {side}: tables differ from _compute_idxs"
        x = np.random.default_rng(1).random((n, 4))
        var = pd.DataFrame(index=[f"g{q}" for q in range(4)])
        ad_host = AnnDataLite(X=x, obsp={"spatial_connectivities": g}, obsm={"spatial": co}, var=var)
        ad_dev = AnnDataLite(X=x, obsp={"spatial_connectivities": g_dev}, obsm={"spatial": co_dev}, var=var)
        frames = [sq.gr.sepal(a, max_neighs=k, n_iter=100, copy=True) for a in (ad_host, ad_dev)] + [sepal_host_tables(ad_host, k)]
        assert all(f.equals(frames[0]) for f in frames[1:]), f"{kind} {side}: sepal frames differ"
        t = median_time({
            "compute_idxs_s": lambda: _compute_idxs(g, co, k),
            "gpu_tables_host_graph_s": lambda: sepal_idxs(g, co, k),
            "gpu_tables_device_graph_s": lambda: sepal_idxs(g_dev, co_dev, k),
            "sepal_host_tables_s": lambda: sepal_host_tables(ad_host, k),
            "sepal_host_graph_s": lambda: sq.gr.sepal(ad_host, max_neighs=k, n_iter=100, copy=True),
            "sepal_device_graph_s": lambda: sq.gr.sepal(ad_dev, max_neighs=k, n_iter=100, copy=True),
        }, sync, args.reps)
        unsat = ref[2]
        is_sat = np.zeros(n, bool)
        is_sat[ref[0]] = True
        orphans = sum(1 for i in unsat if not is_sat[g.indices[g.indptr[i]:g.indptr[i + 1]]].any())
        row = {"lattice": f"{kind} {side}^2, {100 * drop:g} % removed", "spots": n, "unsaturated": int(unsat.size), "orphans": orphans,
               **{name: round(v, 5) for name, v in t.items()}}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del g_dev, co_dev
    res = {"gpu": gpu_info(), "reps": args.reps, "sepal_genes": 4, "sepal_n_iter": 100, "cases": rows}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
