"""The ligrec and sepal calls of ``tests/test_gpu_dist_ligrec_sepal.py``, run on every rank of a process group and once in the
test process without one: host and torch CUDA expression matrices, ``use_raw=True`` for sepal, the permutation counts the test
chooses.  Every input comes from fixed seeds, so every process builds the same data."""

from __future__ import annotations

import numpy as np
import pandas as pd
import scipy.sparse as sp

import squidpy_b200 as sq
from tools import synth

N_CELLS, N_GENES, N_INTER = 1500, 40, 60
SEPAL_GRID = (20, 22)
SEPAL_GENES = 23  # not a multiple of 2 or 3: uneven gene shards


def _ligrec_inputs():
    rng = np.random.default_rng(0)
    x = rng.poisson(0.8, (N_CELLS, N_GENES)).astype(np.float64) * rng.random((N_CELLS, N_GENES)) * 4
    genes = [f"L{i}" for i in range(N_GENES)]
    obs = pd.DataFrame({"cl": pd.Categorical(rng.choice(["t", "b", "m", "n", "e"], N_CELLS))}, index=[f"c{i}" for i in range(N_CELLS)])
    inter = pd.DataFrame({"source": [genes[i] for i in rng.integers(0, N_GENES, N_INTER)],
                          "target": [genes[i] for i in rng.integers(0, N_GENES, N_INTER)]})
    return x, genes, obs, inter


def _sepal_inputs():
    rng = np.random.default_rng(1)
    g, co = synth.hex_graph(*SEPAL_GRID), synth.hex_coords(*SEPAL_GRID)
    n = g.shape[0]
    x = rng.random((n, SEPAL_GENES)) * 3 * (rng.random((n, SEPAL_GENES)) < 0.5)
    x[:, 9] = x[:, 2]  # equal scores: the order of ties follows the gene list
    x[:, 17] = x[:, 2]
    return g, co, x, [f"S{i}" for i in range(SEPAL_GENES)]


def run(perms) -> dict[str, pd.DataFrame]:
    """Every frame of the cases, by name: ligrec's means and p-values from host and device X for each permutation count in
    ``perms``; sepal from host and device X, on all genes, on one gene and with ``use_raw=True``."""
    import torch

    out: dict[str, pd.DataFrame] = {}
    x, genes, obs, inter = _ligrec_inputs()
    for where, X in (("host", x), ("device", torch.as_tensor(x).cuda())):
        ad = sq.AnnDataLite(X=X, obs=obs, var=pd.DataFrame(index=genes), shape=x.shape)
        for p in perms:
            res = sq.gr.ligrec(ad, "cl", interactions=inter, n_perms=int(p), seed=7, copy=True, use_raw=False, threshold=0.05)
            out[f"ligrec/{where}/{p}/means"] = res["means"]
            out[f"ligrec/{where}/{p}/pvalues"] = res["pvalues"]

    g, co, sx, names = _sepal_inputs()
    n = g.shape[0]
    part = np.ascontiguousarray(sx[:, :18])
    for where, X, raw_x in (("host", part, sp.csr_matrix(sx)), ("device", torch.as_tensor(part).cuda(), torch.as_tensor(sx).cuda())):
        raw = sq.AnnDataLite(X=raw_x, obs=pd.DataFrame(index=[f"s{i}" for i in range(n)]), var=pd.DataFrame(index=names), shape=sx.shape)
        ad = sq.AnnDataLite(X=X, obsp={"spatial_connectivities": g}, obsm={"spatial": co}, var=pd.DataFrame(index=names[:18]),
                            raw=raw, shape=(n, 18))
        out[f"sepal/{where}/all"] = sq.gr.sepal(ad, 6, n_iter=3000, copy=True)
        out[f"sepal/{where}/one_gene"] = sq.gr.sepal(ad, 6, genes="S4", n_iter=3000, copy=True)
        out[f"sepal/{where}/raw"] = sq.gr.sepal(ad, 6, genes=names[::-1], use_raw=True, n_iter=3000, copy=True)
    return out
