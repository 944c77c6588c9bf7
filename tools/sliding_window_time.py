"""tl.sliding_window on the GPU at 1 M cells, uniform over a 10 000 x 10 000 square, for the window settings below, against
the same call with the kernel replaced by the numpy restatement ``tests/windows_ref.py`` (frames asserted identical).

    python tools/sliding_window_time.py [--n 1000000] [--reps 3] [--out results.json]

Reports medians of ``--reps`` calls after one warm-up call per setting: the whole call, the kernel time (``ctx.profile``) and
the card with its power limit.  ``reference_cpu_s`` is the unmodified reference (squidpy's per-window pandas masks) timed on a
CPU-only host at the same size; the reference does not run here, so those numbers are quoted, not measured by this script.
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

EXTENT = 10000.0
# name -> (sliding_window kwargs, libraries, reference seconds on a CPU-only host at 1 M cells or None)
SETTINGS = {
    "default": (dict(), 1, 2.3),
    "1000/0": (dict(window_size=1000), 1, 4.0),
    "500/0": (dict(window_size=500), 1, 10.9),
    "2500/500": (dict(window_size=2500, overlap=500), 1, 4.0),
    "1000/0, 2 libraries": (dict(window_size=1000, library_key="library"), 2, None),
}


def make_adata(n: int, n_libs: int = 1, seed: int = 0):
    """n uniform cells over EXTENT^2, obs names cell0.., libraries s0.. interleaved at random."""
    from squidpy_b200 import AnnDataLite

    rng = np.random.default_rng(seed)
    xy = rng.random((n, 2)) * EXTENT
    obs = pd.DataFrame({"library": pd.Categorical.from_codes(rng.integers(0, n_libs, n), categories=[f"s{i}" for i in range(n_libs)])},
                       index=pd.Index([f"cell{i}" for i in range(n)]))
    return AnnDataLite(obs=obs, obsm={"spatial": xy}, shape=(n, 0))


def _card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    args = ap.parse_args()

    import squidpy_b200 as sq
    from squidpy_b200.tl import _sliding_window as swm
    from tests import windows_ref

    ctx = sq.default_context(0)
    gpu_fn = swm.window_ranges
    res = {"card": _card(), "n": args.n, "reps": args.reps, "settings": {}}
    for name, (kw, n_libs, ref_s) in SETTINGS.items():
        adata = make_adata(args.n, n_libs)
        sq.tl.sliding_window(adata, copy=True, **kw)  # warm-up
        t_call, t_kernel = [], []
        for _ in range(args.reps):
            ctx.profile(True)
            ctx.profile_reset()
            # profile mode synchronises every launch; the kernel time is read from this call, the wall time from the next
            sq.tl.sliding_window(adata, copy=True, **kw)
            t_kernel.append(ctx.profile_get("misc")[0])
            ctx.profile(False)
            t0 = time.perf_counter()
            got = sq.tl.sliding_window(adata, copy=True, **kw)
            t_call.append(time.perf_counter() - t0)
        swm.window_ranges = lambda xy, lib, off, s, e, *, ctx=None: windows_ref.window_ranges(xy, lib, off, s, e)
        try:
            exp = sq.tl.sliding_window(adata, copy=True, **kw)
        finally:
            swm.window_ranges = gpu_fn
        pd.testing.assert_frame_equal(got, exp, check_exact=True)
        row = {"columns": got.shape[1], "gpu_call_s": float(np.median(t_call)), "kernel_ms": float(np.median(t_kernel)),
               "reference_cpu_s": ref_s, "equal_to_restatement": True}
        res["settings"][name] = row
        print(name, json.dumps(row), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print("card:", res["card"])


if __name__ == "__main__":
    main()
