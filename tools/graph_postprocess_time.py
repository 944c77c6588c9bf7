"""Wall-clock times of the public post-processors on a caller's graph: the kNN(6) graph of 1M uniform points, built on the GPU
(torch sparse_csr), then ``PercentilePostprocessor(90)`` followed by ``TransformPostprocessor("cosine")`` on the GPU, against
the same two steps in scipy on host copies of the same graph.  ``--steps spectral`` instead times
``TransformPostprocessor("spectral")`` on the same graph with float32 weights, whose column sums depend on the order they are
added in.  The two are run alternately, five times each after a warm-up, and each time ends in a device synchronise; the
outputs are compared entry for entry.  The GPU's name and power limit are read in the same run.  Writes a JSON line to stdout
and to ``--out``.

    python tools/graph_postprocess_time.py --out results/graph_postprocess_time.json
"""

from __future__ import annotations

import argparse
import json
import os
import sys
import time
import warnings

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from squidpy_b200._constants import Transform  # noqa: E402
from squidpy_b200.gr import neighbors as nb  # noqa: E402
from tools.mask_graph_time import gpu_info  # noqa: E402


def main() -> None:
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", choices=["percentile-cosine", "spectral"], default="percentile-cosine")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    co = np.random.default_rng(0).uniform(0, 1000, (args.n, 2))
    adj, dst = nb.KNNBuilder(n_neighs=6).build(torch.tensor(co, device="cuda"))
    if args.steps == "spectral":
        w = torch.rand(adj.values().numel(), generator=torch.Generator().manual_seed(1)).add_(0.05).cuda()
        adj = torch.sparse_csr_tensor(adj.crow_indices(), adj.col_indices(), w, size=adj.shape)
    to_host = lambda t: sp.csr_matrix((t.values().cpu().numpy(), t.col_indices().cpu().numpy(), t.crow_indices().cpu().numpy()), shape=tuple(t.shape))
    hadj, hdst = to_host(adj), to_host(dst)
    steps = ([nb.TransformPostprocessor(Transform.SPECTRAL)] if args.steps == "spectral"
             else [nb.PercentilePostprocessor(90.0), nb.TransformPostprocessor(Transform.COSINE)])

    def run(a, d):
        for s in steps:
            a, d = s(a, d)
        return a, d

    def timed(fn):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    warnings.simplefilter("ignore", sp.SparseEfficiencyWarning)
    timed(lambda: run(adj, dst))
    dev_t, host_t = [], []
    for _ in range(args.reps):
        t, (da, dd) = timed(lambda: run(adj, dst))
        dev_t.append(t)
        t, (ha, hd) = timed(lambda: run(hadj.copy(), hdst.copy()))
        host_t.append(t)
    same = True
    for got, want in ((to_host(da), sp.csr_matrix(ha)), (to_host(dd), sp.csr_matrix(hd))):
        want.sort_indices()
        same &= bool(np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
                     and np.array_equal(got.data.view(np.uint8), want.data.view(np.uint8)))
    rec = {"gpu": gpu_info(), "n": args.n, "graph": "kNN(6), device-built", "steps": "spectral, float32 weights" if args.steps == "spectral" else "percentile(90) + cosine", "nnz": int(adj.values().numel()),
           "device_s_median": float(np.median(dev_t)), "device_s": dev_t, "scipy_host_s_median": float(np.median(host_t)), "scipy_host_s": host_t,
           "equal_bit_for_bit": same}
    line = json.dumps(rec)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
