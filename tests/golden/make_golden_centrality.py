"""Generates tests/golden/centrality.npz: the UNMODIFIED reference ``centrality_scores`` (the squidpy source tree named by
``$SQUIDPY_REF``, through the stub-import loader ``oracle/_refload.py``).  Only runnable where the reference tree exists; the output is
committed.

    python tests/golden/make_golden_centrality.py

rustworkx is not installed here.  The reference's graph calls go to a test-only shim (``PyGraph``,
``group_closeness_centrality``, ``group_degree_centrality``) backed by networkx, which the reference's own parity test
(``tests/graph/test_nhood.py:91-105``) pins them to.  Where networkx raises because the measure is undefined — closeness
of an empty group, degree of a group holding every node — the shim returns NaN, the value this library documents.  Like rustworkx, the shim returns a
float: networkx gives the int 0 for a closeness sum of 0.

Fixtures: a hexagonal lattice, a directed kNN graph and a radius graph (with isolated points and several components), a
hand-made graph with self loops, explicit zeros and a cancelling pair in every value dtype, non-canonical CSR (duplicates),
NaN labels, an unused category, one category, and 63, 64, 65 and 130 categories.  Per case: every single score and
``score=None``.  Then the reference's errors, type and message.
"""

from __future__ import annotations

import math
import os
import sys

import numpy as np
import pandas as pd
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from squidpy_b200._adata import AnnDataLite  # noqa: E402
from tools import synth  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
SCORES = [None, "degree_centrality", "average_clustering", "closeness_centrality"]


def _knn(xy, k):
    from sklearn.neighbors import NearestNeighbors

    return NearestNeighbors(n_neighbors=k).fit(xy).kneighbors_graph(mode="connectivity").tocsr()  # directed, float64 ones


def _radius(xy, r):
    from sklearn.neighbors import radius_neighbors_graph

    return radius_neighbors_graph(xy, r, mode="connectivity", include_self=True).tocsr()  # self loops on the diagonal


def _handmade(dtype):
    """Two components with a self loop, an explicit zero, a cancelling pair and a duplicate-free triangle, plus isolated
    nodes 9 and 10.  Integer values that cancel only after wrapping at the dtype's width: 100 + 156 = 0 in uint8,
    -128 + -128 = 0 in int8."""
    n = 11
    ent = {(0, 1): 1, (1, 0): 1, (1, 2): 2, (2, 0): 3, (0, 0): 5, (2, 3): 0, (3, 4): 7, (4, 3): -7, (4, 5): 1, (5, 6): 1, (6, 4): 1,
           (7, 8): 1, (8, 7): 1, (6, 7): 2}
    if dtype == np.uint8:
        ent[(3, 4)], ent[(4, 3)] = 100, 156
    if dtype == np.int8:
        ent[(3, 4)], ent[(4, 3)] = -128, -128
    if dtype == np.bool_:
        ent = {k: v != 0 for k, v in ent.items()}
    r, c = np.array(list(ent)).T
    v = np.array([ent[k] for k in ent]).astype(dtype) if dtype != np.uint8 else np.array([ent[k] % 256 for k in ent], dtype=np.uint8)
    return sp.csr_matrix((v, (r, c)), shape=(n, n))


def _duplicates(float_vals: bool):
    """A non-canonical CSR: (0, 1) stored twice summing to zero against (1, 0), (2, 3) stored twice, unsorted rows."""
    indptr = np.array([0, 3, 4, 6, 7, 7], dtype=np.int32)
    indices = np.array([1, 4, 1, 0, 3, 3, 2], dtype=np.int32)
    data = np.array([2, 1, 1, -3, 1, 1, 1], dtype=np.float64 if float_vals else np.int64)
    return sp.csr_matrix((data, indices, indptr), shape=(5, 5))


def _labels(n, n_cls, seed, nan_frac=0.0):
    rng = np.random.default_rng(seed)
    codes = rng.integers(0, n_cls, n)
    if nan_frac:
        codes[rng.random(n) < nan_frac] = -1
    return codes


def cases():
    """(name, graph, codes, n_categories)."""
    rng = np.random.default_rng(0)
    hexg = synth.hex_graph(12, 10)
    out = [("hex", hexg, _labels(120, 5, 1), 5),
           ("hex_nan_unused", hexg, np.where(_labels(120, 4, 2, 0.1) == 3, 4, _labels(120, 4, 2, 0.1)), 6)]
    xy = rng.random((150, 2)) * 100
    out.append(("knn_directed", _knn(xy, 4), _labels(150, 7, 3), 7))
    xy2 = np.concatenate([rng.random((100, 2)) * 60, rng.random((20, 2)) * 60 + 200, [[500.0, 500.0], [-300.0, 0.0]]])
    out.append(("radius_components", _radius(xy2, 9.0), _labels(122, 4, 4, 0.05), 4))
    for dt in (np.float64, np.float32, np.int64, np.int32, np.int16, np.int8, np.uint8, np.uint32, np.uint64, np.bool_):
        out.append((f"handmade_{np.dtype(dt).name}", _handmade(dt), np.array([0, 0, 1, 1, 2, 2, 2, 0, 1, -1, 2]), 4))
    out.append(("duplicates_float", _duplicates(True), np.array([0, 1, 0, 1, 1]), 2))
    out.append(("duplicates_int", _duplicates(False), np.array([0, 1, 0, 1, 1]), 2))
    out.append(("one_category", hexg, np.zeros(120, dtype=np.int64), 1))
    out.append(("one_category_nan", hexg, np.where(_labels(120, 2, 5) == 1, -1, 0), 1))
    xy3 = rng.random((400, 2)) * 100
    g3 = _knn(xy3, 5)
    for k in (63, 64, 65, 130):
        out.append((f"cats{k}", g3, _labels(400, k, k), k))
    out.append(("csc_input", _knn(xy, 3).tocsc(), _labels(150, 3, 6), 3))
    return out


def make_adata(graph, codes, n_cls):
    cats = [f"c{i}" for i in range(n_cls)]
    obs = pd.DataFrame({"cluster": pd.Categorical.from_codes(np.asarray(codes), categories=cats)},
                       index=[str(i) for i in range(len(codes))])
    return AnnDataLite(X=np.zeros((len(codes), 1)), obs=obs, var=pd.DataFrame(index=["g0"]), obsp={"spatial_connectivities": graph})


def error_cases(graph, codes):
    """(name, adata factory, kwargs) of calls the reference refuses."""
    def base():
        return make_adata(graph, codes, 3)

    def numeric():
        a = base()
        a.obs["num"] = np.arange(len(codes))
        return a

    return [("score_list", base, dict(cluster_key="cluster", score=["degree_centrality"])),
            ("score_int", base, dict(cluster_key="cluster", score=3)),
            ("score_invalid", base, dict(cluster_key="cluster", score="betweenness")),
            ("missing_cluster_key", base, dict(cluster_key="nope")),
            ("non_categorical", numeric, dict(cluster_key="num")),
            ("missing_connectivity", base, dict(cluster_key="cluster", connectivity_key="other"))]


def install_rustworkx_shim():
    """rustworkx's graph calls of the reference, on networkx (test only)."""
    import networkx as nx

    rx = sys.modules["rustworkx"]

    class PyGraph:
        def __init__(self, multigraph=False):
            self.g = nx.Graph()

        def add_nodes_from(self, nodes):
            self.g.add_nodes_from(nodes)

        def add_edges_from_no_data(self, edges):
            self.g.add_edges_from(edges)

    def group_closeness_centrality(graph, idx):
        idx = [int(i) for i in idx]
        return math.nan if not idx else float(nx.group_closeness_centrality(graph.g, idx))

    def group_degree_centrality(graph, idx):
        idx = [int(i) for i in idx]
        return math.nan if len(idx) == graph.g.number_of_nodes() else float(nx.group_degree_centrality(graph.g, idx))

    rx.PyGraph = PyGraph
    rx.group_closeness_centrality = group_closeness_centrality
    rx.group_degree_centrality = group_degree_centrality


def main():
    import networkx as nx

    from oracle import _refload

    nh = _refload.load()["nh"]
    install_rustworkx_shim()
    out = {"meta": np.array(f"numpy {np.__version__}; pandas {pd.__version__}; networkx {nx.__version__}; reference squidpy "
                            "centrality_scores with a networkx-backed rustworkx shim")}
    all_cases = cases()
    for i, (name, g, codes, n_cls) in enumerate(all_cases):
        out[f"c{i}_name"] = np.array(name)
        out[f"c{i}_format"] = np.array(g.format)
        out[f"c{i}_indptr"], out[f"c{i}_indices"], out[f"c{i}_data"] = g.indptr, g.indices, g.data
        out[f"c{i}_codes"], out[f"c{i}_ncls"] = np.asarray(codes, dtype=np.int64), np.array(n_cls)
        for j, score in enumerate(SCORES):
            df = nh.centrality_scores(make_adata(g, codes, n_cls), "cluster", score=score, copy=True)
            assert list(df.index) == [f"c{k}" for k in range(n_cls)]
            out[f"c{i}_s{j}_cols"] = np.array(list(df.columns))
            out[f"c{i}_s{j}_values"] = df.to_numpy()
            out[f"c{i}_s{j}_dtypes"] = np.array([str(t) for t in df.dtypes])
        a = make_adata(g, codes, n_cls)
        nh.centrality_scores(a, "cluster")
        stored = a.uns["cluster_centrality_scores"]
        np.testing.assert_array_equal(stored.to_numpy(), out[f"c{i}_s0_values"])
    g0, codes0 = synth.hex_graph(4, 4), _labels(16, 3, 9)
    for j, (name, factory, kw) in enumerate(error_cases(g0, codes0)):
        try:
            nh.centrality_scores(factory(), copy=True, **kw)
        except Exception as e:  # noqa: BLE001
            out[f"e{j}_name"], out[f"e{j}_type"], out[f"e{j}_msg"] = np.array(name), np.array(type(e).__name__), np.array(str(e))
        else:
            raise AssertionError(f"{name}: the reference did not raise")
    np.savez_compressed(os.path.join(OUT, "centrality.npz"), **out)
    print("wrote centrality.npz:", len(all_cases), "cases,", len(error_cases(g0, codes0)), "error cases")


if __name__ == "__main__":
    main()
