"""The calculate_niche embeddings on the GPU against the same embeddings computed on the host with scipy, the way the
reference computes them, on the same data.

Legs (each: medians of ``--reps`` alternated device / host calls after one warm-up of each):
  * neighbourhood profile, 1 M-spot hex lattice, 20 categories, distance 3: ``niche_profile`` against powers of A by scipy
    SpGEMM and per-category column sums of each (``_calculate_neighborhood_profile``'s computation, without its LIL writes);
  * UTAG, 200 000 cells x 300 genes (CSR, 10 %): ``niche_aggregate(..., "utag")`` against ``normalize(A, "l1") @ X``;
  * CellCharter mean, the same data, distance 3: ``niche_aggregate(..., "mean", 3)`` against the reference's hop recursion,
    normalisation and aggregation on scipy (``tests/niche_ref.py``).
  * CellCharter mean on a 1 M-cell kNN graph with 15 neighbours, 8 genes, distance 3: device only, the case whose hop rows
    exceed the shared-memory tables and run from global-memory tables in batches.
Outputs are compared: profiles and UTAG bit for bit, CellCharter within 1e-12 relative.  Prints the card and its power limit;
``--out FILE`` also writes the results as JSON.

    python tools/niche_time.py [--reps 3] [--out FILE]
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
from squidpy_b200.gr import niche_aggregate, niche_profile  # noqa: E402
from tests import niche_ref  # noqa: E402
from tools import synth  # noqa: E402


def host_profile(A, codes, n_cls, distance):
    """Column sums of A, A^2, ... per category (the reference's profile computation), proportions, equal weights."""
    members = [np.flatnonzero(codes == c) for c in range(n_cls)]
    Ak, out = A, None
    for k in range(distance):
        if k:
            Ak = Ak @ A
        csc = Ak.tocsc()
        P = np.column_stack([np.asarray(csc[:, m].sum(axis=1)).ravel() for m in members]).astype(np.float64)
        t = P.sum(axis=1)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = np.nan_to_num(P / t[:, None], nan=0.0)
        out = q if out is None else out + q
    return out / distance


def timed(f):
    t = time.perf_counter()
    r = f()
    return time.perf_counter() - t, r


def leg(name, dev, host, reps, check):
    dev(), host()
    td, th = [], []
    for _ in range(reps):
        t, rd = timed(dev)
        td.append(t)
        t, rh = timed(host)
        th.append(t)
    check(rd, rh)
    res = {"leg": name, "device_s": float(np.median(td)), "host_s": float(np.median(th))}
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card, flush=True)
    rng = np.random.default_rng(0)
    results = []
    A = synth.hex_graph(1000, 1000)
    codes = rng.integers(0, 20, A.shape[0]).astype(np.int32)
    results.append(leg("profile 1M hex, 20 categories, distance 3", lambda: niche_profile(A, codes, 20, 3),
                       lambda: host_profile(A, codes, 20, 3), args.reps, lambda d, h: np.testing.assert_allclose(d, h, rtol=1e-12)))
    B = synth.hex_graph(400, 500)
    X = sp.random(B.shape[0], 300, density=0.1, format="csr", dtype=np.float32, random_state=1)
    X.data = np.floor(X.data * 8).astype(np.float32)
    results.append(leg("utag 200k x 300, CSR 10%", lambda: niche_aggregate(B, X, "utag")[0], lambda: niche_ref.utag(B, X), args.reps,
                       np.testing.assert_array_equal))
    results.append(leg("cellcharter mean 200k x 300, CSR 10%, distance 3", lambda: niche_aggregate(B, X, "mean", 3)[0],
                       lambda: niche_ref.cellcharter(B, X, 3, "mean")[0], args.reps, lambda d, h: np.testing.assert_allclose(d, h, rtol=1e-12)))
    # many long rows: a 1 M-cell kNN graph with 15 neighbours at distance 3 (hop-3 bounds in the thousands), device only
    from squidpy_b200.gr import knn_2d

    n = 1_000_000
    _, idx = knn_2d(rng.random((n, 2)) * 1000, 15)
    K = sp.csr_matrix((np.ones(idx.size, np.float32), idx.ravel(), np.arange(0, idx.size + 1, 15)), shape=(n, n))
    Xk = sp.random(n, 8, density=0.3, format="csr", dtype=np.float32, random_state=3)
    niche_aggregate(K, Xk, "mean", 3)
    t = []
    for _ in range(args.reps):
        dt, (_, hop_nnz) = timed(lambda: niche_aggregate(K, Xk, "mean", 3))
        t.append(dt)
    res = {"leg": "cellcharter mean 1M kNN(15) x 8, distance 3 (host not run)", "device_s": float(np.median(t)), "hop_nnz": hop_nnz.tolist()}
    print(json.dumps(res), flush=True)
    results.append(res)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"card": card, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
