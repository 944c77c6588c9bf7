"""Generates tests/golden/niche.npz: the UNMODIFIED reference niche calling (``src/squidpy/gr/_niche.py`` of the squidpy tree
named by ``$SQUIDPY_REF``, through the stub-import loader ``oracle/_refload.py``).  Only runnable where the reference tree
exists; the output is committed.

    python tests/golden/make_golden_niche.py

anndata and scanpy are not installed here.  ``anndata.AnnData`` is bound to ``AnnDataLite`` and scanpy to the recording
stand-in ``tests/niche_scanpy_standin.py``, so the golden holds every matrix the reference hands to scanpy and the ``obs``
columns it ends with; scikit-learn's GaussianMixture is the real one.

Cases (``cases()``, shared with the tests): a hex lattice, a directed kNN graph, a radius graph with isolated cells and self
loops, a non-canonical graph with explicit zeros and duplicates, a float-weighted graph, a CSC graph and an int64-weighted
graph; NaN labels and an
unused category; distance 1-4 with short ``n_hop_weights``, ``abs_nhood`` and ``scale`` both ways; sparse and dense X (CellCharter
without ``use_rep`` fails on a dense X in the reference, both ways: an error case), mean and variance; ``use_rep``; ``mask``, ``min_niche_size`` and ``library_key`` with three libraries.  Then the reference's errors and
warnings, type and message.
"""

from __future__ import annotations

import json
import logging
import os
import sys
import warnings

import numpy as np
import pandas as pd
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from squidpy_b200._adata import AnnDataLite  # noqa: E402
from tests import niche_scanpy_standin as standin  # noqa: E402
from tools import synth  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def _knn(xy, k):
    from sklearn.neighbors import NearestNeighbors

    return NearestNeighbors(n_neighbors=k).fit(xy).kneighbors_graph(mode="connectivity").tocsr()


def _radius(xy, r):
    from sklearn.neighbors import radius_neighbors_graph

    return radius_neighbors_graph(xy, r, mode="connectivity", include_self=True).tocsr().astype(np.float32)


def graphs() -> dict[str, sp.spmatrix]:
    rng = np.random.default_rng(0)
    out = {"hex": synth.hex_graph(12, 10)}
    out["knn"] = _knn(rng.random((120, 2)) * 100, 5)
    xy = np.concatenate([rng.random((110, 2)) * 60, rng.random((8, 2)) * 60 + 200, [[500.0, 500.0], [-300.0, 0.0]]])
    out["radius"] = _radius(xy, 9.0)
    h = synth.hex_graph(12, 10).tocoo()
    extra = rng.integers(0, h.nnz, 40)
    r = np.concatenate([h.row, h.row[extra], [0, 5, 7]])
    c = np.concatenate([h.col, h.col[extra], [0, 5, 9]])
    v = np.concatenate([h.data, h.data[extra], [0.0, 1.0, 0.0]]).astype(np.float32)
    perm = rng.permutation(r.size)
    order = np.argsort(r[perm], kind="stable")
    noncanon = sp.csr_matrix((v[perm][order], c[perm][order], np.concatenate([[0], np.cumsum(np.bincount(r, minlength=120))])), shape=h.shape)
    out["noncanonical"] = noncanon
    w = synth.hex_graph(12, 10)
    w.data = (rng.random(w.nnz) * 1.5 + 0.25).astype(np.float32)
    out["weighted"] = w
    out["csc"] = _knn(rng.random((120, 2)) * 100, 4).astype(np.float32).tocsc()
    iw = synth.hex_graph(12, 10).astype(np.int64)
    iw.data = rng.integers(1, 4, iw.nnz).astype(np.int64)
    out["int64"] = iw
    return out


def make_adata(graph, seed=0, n_cls=5, nan_frac=0.05, sparse_x=True, x_dtype=np.float32, n_genes=12, libs=False):
    n = graph.shape[0]
    rng = np.random.default_rng(seed)
    codes = rng.integers(0, n_cls, n)
    codes[rng.random(n) < nan_frac] = -1
    cats = [f"t{i}" for i in range(n_cls + 1)]  # the last category is never used
    obs = pd.DataFrame({"cell_type": pd.Categorical.from_codes(codes, categories=cats)}, index=[f"cell{i}" for i in range(n)])
    if libs:
        obs["library"] = pd.Categorical(np.array(["a", "b", "c"])[np.arange(n) * 3 // n])
    X = np.floor(rng.exponential(2.0, (n, n_genes)) * (rng.random((n, n_genes)) < 0.3)).astype(x_dtype)
    if sparse_x:
        X = sp.csr_matrix(X)
    rep = rng.normal(size=(n, 6))
    return AnnDataLite(X=X, obs=obs, var=pd.DataFrame(index=[f"g{i}" for i in range(n_genes)]), obsp={"spatial_connectivities": graph.copy()},
                       obsm={"X_rep": rep})


def cases() -> list[tuple[str, str, dict, dict]]:
    """(name, function, adata kwargs, call kwargs) for every golden call; the graph is named by adata kwargs["graph"]."""
    out = []
    for g in ("hex", "knn", "radius", "noncanonical", "weighted", "csc", "int64"):
        out.append((f"nh_{g}_d1", "neighborhood", dict(graph=g), dict(groups="cell_type", resolutions=[0.5, 1.0], n_neighbors=10)))
        out.append((f"nh_{g}_d3", "neighborhood", dict(graph=g, seed=1),
                    dict(groups="cell_type", resolutions=0.5, distance=3, n_hop_weights=[1.0, 0.5])))
        out.append((f"utag_{g}_sparse", "utag", dict(graph=g), dict(resolutions=[0.5])))
        out.append((f"cc_{g}_mean_d3", "cellcharter", dict(graph=g), dict(distance=3, aggregation="mean", n_components=4)))
    out += [
        ("nh_hex_d2_abs", "neighborhood", dict(graph="hex", seed=2), dict(groups="cell_type", resolutions=0.5, distance=2, abs_nhood=True)),
        ("nh_hex_d4_noscale", "neighborhood", dict(graph="hex", seed=3),
         dict(groups="cell_type", resolutions=[0.3], distance=4, scale=False, n_hop_weights=[2, 1, 0.5, 0.25, 9.0])),
        ("nh_radius_d2_abs_noscale", "neighborhood", dict(graph="radius"), dict(groups="cell_type", resolutions=0.5, distance=2,
                                                                               abs_nhood=True, scale=False)),
        ("utag_hex_dense32", "utag", dict(graph="hex", sparse_x=False), dict(resolutions=0.5)),
        ("utag_knn_dense64", "utag", dict(graph="knn", sparse_x=False, x_dtype=np.float64), dict(resolutions=0.5)),
        ("cc_hex_var_d2", "cellcharter", dict(graph="hex"), dict(distance=2, aggregation="variance", n_components=3)),
        ("cc_radius_var_d4", "cellcharter", dict(graph="radius"), dict(distance=4, aggregation="variance", n_components=3)),
        ("cc_knn_d1", "cellcharter", dict(graph="knn"), dict(distance=1, aggregation="mean", n_components=3)),
        ("cc_hex_sparse64_d2", "cellcharter", dict(graph="hex", x_dtype=np.float64), dict(distance=2, n_components=3)),
        ("cc_use_rep", "cellcharter", dict(graph="hex"), dict(use_rep="X_rep", n_components=4)),
        ("nh_mask_min_size", "neighborhood", dict(graph="hex"), dict(groups="cell_type", resolutions=[0.5, 1.0], min_niche_size=12,
                                                                     mask="every_third")),
        ("nh_library", "neighborhood", dict(graph="hex", libs=True), dict(groups="cell_type", resolutions=0.5, distance=2,
                                                                          library_key="library", min_niche_size=3)),
        ("utag_library_mask", "utag", dict(graph="knn", libs=True), dict(resolutions=[0.5], library_key="library", mask="every_third")),
        ("cc_library", "cellcharter", dict(graph="hex", libs=True), dict(distance=2, n_components=3, library_key="library", inplace=False)),
        ("dispatch_nh", "calculate_niche", dict(graph="hex"), dict(flavor="neighborhood", groups="cell_type", n_neighbors=10, distance=2,
                                                                            resolutions=[0.5])),
        ("dispatch_cc", "calculate_niche", dict(graph="knn"), dict(flavor="cellcharter", n_components=3)),
    ]
    return out


def build_call(case, graphs_):
    """(adata, kwargs) of one case, the mask resolved against the adata."""
    name, fn, akw, kw = case
    akw = dict(akw)
    adata = make_adata(graphs_[akw.pop("graph")], **akw)
    kw = dict(kw)
    if kw.get("mask") == "every_third":
        kw["mask"] = pd.Series(np.arange(adata.n_obs) % 3 != 0, index=adata.obs.index)
    return adata, kw


def error_cases() -> list[tuple[str, dict]]:
    """calculate_niche calls the reference refuses (on the hex adata)."""
    return [
        ("bad_flavor", dict(flavor="kmeans", groups="cell_type", n_neighbors=10)),
        ("missing_groups", dict(flavor="neighborhood", n_neighbors=10)),
        ("missing_n_neighbors", dict(flavor="utag")),
        ("missing_resolutions", dict(flavor="utag", n_neighbors=10)),
        ("bad_library_key", dict(flavor="utag", n_neighbors=10, library_key="nope")),
        ("library_key_type", dict(flavor="utag", n_neighbors=10, library_key=3)),
        ("n_neighbors_type", dict(flavor="utag", n_neighbors=10.0)),
        ("resolutions_type", dict(flavor="utag", n_neighbors=10, resolutions=1)),
        ("resolutions_tuple", dict(flavor="utag", n_neighbors=10, resolutions=(0.5, 1))),
        ("resolutions_list", dict(flavor="utag", n_neighbors=10, resolutions=[0.5, "a"])),
        ("n_hop_weights_type", dict(flavor="neighborhood", groups="cell_type", n_neighbors=10, n_hop_weights=(1.0,))),
        ("scale_type", dict(flavor="neighborhood", groups="cell_type", n_neighbors=10, scale=1)),
        ("abs_nhood_type", dict(flavor="neighborhood", groups="cell_type", n_neighbors=10, abs_nhood=0)),
        ("groups_type", dict(flavor="neighborhood", groups=3, n_neighbors=10)),
        ("min_size_type", dict(flavor="neighborhood", groups="cell_type", n_neighbors=10, min_niche_size=2.0)),
        ("distance_zero", dict(flavor="neighborhood", groups="cell_type", n_neighbors=10, distance=0)),
        ("cc_distance_type", dict(flavor="cellcharter", distance=2.0)),
        ("cc_distance_zero", dict(flavor="cellcharter", distance=0)),
        ("cc_aggregation", dict(flavor="cellcharter", aggregation="max")),
        ("cc_aggregation_type", dict(flavor="cellcharter", aggregation=1)),
        ("cc_n_components", dict(flavor="cellcharter", n_components=0)),
        ("cc_n_components_type", dict(flavor="cellcharter", n_components=2.0)),
        ("cc_random_state_type", dict(flavor="cellcharter", random_state=1.0)),
        ("cc_use_rep_type", dict(flavor="cellcharter", use_rep=3)),
        ("inplace_type", dict(flavor="utag", n_neighbors=10, inplace=1)),
        ("cc_dense_variance", dict(flavor="cellcharter", aggregation="variance", n_components=3, distance=1)),
        ("cc_dense_mean", dict(flavor="cellcharter", aggregation="mean", n_components=3, distance=2)),
        ("cc_use_rep_short", dict(flavor="cellcharter", use_rep="X_rep", n_components=8)),
        ("cc_use_rep_missing", dict(flavor="cellcharter", use_rep="nope", n_components=3)),
    ]


def warning_cases() -> list[tuple[str, dict]]:
    """calculate_niche calls that log "not used" warnings (captured as log records)."""
    return [
        ("utag_unused", dict(flavor="utag", n_neighbors=10, resolutions=[0.5], groups="cell_type", distance=2, scale=False, abs_nhood=True, random_state=1)),
        ("nh_unused", dict(flavor="neighborhood", groups="cell_type", n_neighbors=10, resolutions=0.5, aggregation="mean", n_components=3, use_rep="X_rep")),
        ("cc_unused", dict(flavor="cellcharter", n_components=3, groups="cell_type", n_neighbors=10, resolutions=[0.5], min_niche_size=2,
                           n_hop_weights=[1.0])),
    ]


class _Records(logging.Handler):
    def __init__(self):
        super().__init__()
        self.records: list[str] = []

    def emit(self, record):
        self.records.append(f"{record.levelname}:{record.getMessage()}")


def load_reference():
    from oracle import _refload

    _refload.load()
    sys.modules["anndata"].AnnData = AnnDataLite
    _refload._stub("spatialdata", SpatialData=sys.modules["spatialdata"].SpatialData, sanitize_table=lambda a: None)
    _refload._stub("spatialdata._logging", logger=logging.getLogger("squidpy_ref_niche"))
    import importlib

    ref = importlib.import_module("squidpy.gr._niche")
    ref.sc = standin.install()
    return ref


def run(fn_module, fn, adata, kw):
    """Calls ``fn`` of ``fn_module`` (the reference or this library) on ``adata``; returns (adata holding the result, calls)."""
    standin.CALLS.clear()
    f = getattr(fn_module, fn if fn == "calculate_niche" else f"calculate_niche_{fn}")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        res = f(adata, **kw)
    return (adata if res is None else res), list(standin.CALLS)


def main():
    ref = load_reference()
    gs = graphs()
    out = {"meta": np.array(f"numpy {np.__version__}; pandas {pd.__version__}; reference squidpy calculate_niche_* with the scanpy stand-in")}
    for i, case in enumerate(cases()):
        adata, kw = build_call(case, gs)
        before = set(adata.obs.columns)
        res, calls = run(ref, case[1], adata, kw)
        out[f"c{i}_name"] = np.array(case[0])
        out[f"c{i}_ncalls"] = np.array(len(calls))
        for j, (cname, X, info) in enumerate(calls):
            out[f"c{i}_k{j}_name"] = np.array(cname)
            out[f"c{i}_k{j}_X"] = X
            out[f"c{i}_k{j}_info"] = np.array(json.dumps(info, sort_keys=True))
        cols = sorted(set(res.obs.columns) - before)
        out[f"c{i}_cols"] = np.array(cols)
        for j, col in enumerate(cols):
            out[f"c{i}_col{j}"] = np.array(res.obs[col].astype(str).to_numpy(), dtype=str)
    hexg = gs["hex"]
    for j, (name, kw) in enumerate(error_cases()):
        adata = make_adata(hexg, sparse_x=not name.startswith("cc_dense"))
        try:
            run(ref, "calculate_niche", adata, kw)
        except Exception as e:  # noqa: BLE001
            out[f"e{j}_name"], out[f"e{j}_type"], out[f"e{j}_msg"] = np.array(name), np.array(type(e).__name__), np.array(str(e))
        else:
            raise AssertionError(f"{name}: the reference did not raise")
    logger = logging.getLogger("squidpy_ref_niche")
    for j, (name, kw) in enumerate(warning_cases()):
        h = _Records()
        logger.addHandler(h)
        logger.setLevel(logging.DEBUG)
        with warnings.catch_warnings(record=True) as ws:
            warnings.simplefilter("always")
            ref.calculate_niche(make_adata(hexg), **kw)
        logger.removeHandler(h)
        out[f"w{j}_name"] = np.array(name)
        out[f"w{j}_log"] = np.array([r for r in h.records if r.startswith("WARNING")], dtype=str)
        out[f"w{j}_warn"] = np.array([f"{w.category.__name__}:{w.message}" for w in ws], dtype=str)
    np.savez_compressed(os.path.join(OUT, "niche.npz"), **out)
    print("wrote niche.npz:", len(cases()), "cases,", len(error_cases()), "error cases,", len(warning_cases()), "warning cases")


if __name__ == "__main__":
    main()
