"""Writes ``tests/golden/postprocessors.npz``: the output of the UNMODIFIED reference post-processors
(``DistanceIntervalPostprocessor``, ``PercentilePostprocessor``, ``TransformPostprocessor``), of ``GraphBuilderCSR.combine`` and
of ``_resolve_graph_builder`` (``squidpy/gr/neighbors.py``, ``squidpy/gr/_build.py``), run through ``oracle/_refload.py``.

    python tests/golden/make_golden_postprocessors.py

Cases (``pp/<case>/...``): seeded graph pairs with ``adj`` and ``dst`` of different sparsity patterns, explicit zeros, empty
rows, float32 and float64 ``dst``, weighted ``adj``, interval bounds between float32 neighbours, percentiles at 0, 100 and
between tied values, and two- and three-step chains.  Every input and output is stored as CSR arrays (outputs after
``sort_indices()``), with the chain as JSON; a chain the reference refuses stores the exception's type instead.  Spectral is
left out: the reference sums degrees with ``fast_array_utils``, which is not installed here.  ``combine/<case>/...`` holds
library blocks and their (interleaved) observation indices.  ``resolve/<i>`` holds the builder ``_resolve_graph_builder``
returns for a grid of arguments (class, ``uns_params``, post-processors, warnings) or its error.  ``known/...`` holds the known
answers of the reference's ``tests/graph/test_spatial_neighbors.py`` as data: the Visium fixture's coordinates with its
ring sums 6 / 18 / 36 and distance sums 0 / 30 / 84 of row 0, and the square-grid fixture with maximum degrees 4 / 12 / 24.
"""

from __future__ import annotations

import importlib
import itertools
import json
import os
import sys
import types
import warnings

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "postprocessors.npz")


def _reference():
    """(neighbors module, _build module, logged warnings) of the reference; ``gr/_build.py`` needs a few more stubs than
    ``oracle/_refload.py`` registers (geopandas, shapely and the spatialdata internals it imports)."""
    sys.path.insert(0, ROOT)
    from oracle import _refload

    mods = _refload.load()
    logged: list[str] = []

    class _Logger:
        @staticmethod
        def warning(msg, *a, **k):
            logged.append(str(msg))

        @staticmethod
        def info(*a, **k):
            return None

        debug = error = info

    def stub(name, **attrs):
        m = sys.modules.get(name) or types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m

    anything = type("Anything", (), {"__init__": lambda self, *a, **k: None})
    stub("geopandas")
    stub("shapely", LineString=anything, MultiPolygon=anything, Polygon=anything)
    stub("spatialdata", SpatialData=anything)
    stub("spatialdata._core")
    stub("spatialdata._core.centroids", get_centroids=None)
    stub("spatialdata._core.query")
    stub("spatialdata._core.query.relational_query", get_element_instances=None, match_element_to_table=None)
    stub("spatialdata._logging", logger=_Logger)
    stub("spatialdata.models", get_table_keys=None, Labels2DModel=anything, Labels3DModel=anything, get_model=None)
    stub("spatialdata.models.models", Labels2DModel=anything, Labels3DModel=anything, get_model=None)
    build = importlib.import_module("squidpy.gr._build")
    return mods["nb"], build, logged


def _put(out: dict, prefix: str, m) -> None:
    m = sp.csr_matrix(m)
    m.sort_indices()
    out[f"{prefix}/indptr"] = np.asarray(m.indptr, dtype=np.int64)
    out[f"{prefix}/indices"] = np.asarray(m.indices, dtype=np.int64)
    out[f"{prefix}/data"] = m.data.copy()
    out[f"{prefix}/n"] = np.int64(m.shape[0])


def _csr(rows: list[list[tuple[int, float]]], n: int, dtype) -> sp.csr_matrix:
    indptr = np.zeros(n + 1, dtype=np.int32)
    indptr[1:] = np.cumsum([len(r) for r in rows])
    idx = np.array([j for r in rows for j, _ in r], dtype=np.int32)
    val = np.array([v for r in rows for _, v in r], dtype=dtype)
    m = sp.csr_matrix((val, idx, indptr), shape=(n, n))
    m.has_sorted_indices = True
    return m


def _pair(rng, n: int, *, same: bool, dst_dtype, weighted: bool = False, zeros: int = 0, empty: int = 0, ties: bool = False, p: float = 0.25):
    """(adj float32, dst) of n x n with sorted columns: the same pattern or independent ones, ``zeros`` explicit zeros in
    each, ``empty`` empty rows, tied integer distances with ``ties``."""
    dead = set(rng.choice(n, size=empty, replace=False).tolist()) if empty else set()

    def pattern():
        return [[] if i in dead else sorted(rng.choice(n, size=rng.binomial(n, p), replace=False).tolist()) for i in range(n)]

    pa = pattern()
    pd_ = pa if same else pattern()
    a_rows = [[(j, float(rng.uniform(0.25, 2.0)) if weighted else 1.0) for j in r] for r in pa]
    d_rows = [[(j, float(rng.integers(1, 5)) if ties else float(rng.uniform(0.5, 10.0))) for j in r] for r in pd_]
    for rows in (a_rows, d_rows):
        flat = [(i, t) for i, r in enumerate(rows) for t in range(len(r))]
        for k in rng.choice(len(flat), size=min(zeros, len(flat)), replace=False) if flat else []:
            i, t = flat[k]
            rows[i][t] = (rows[i][t][0], 0.0)
    return _csr(a_rows, n, np.float32), _csr(d_rows, n, dst_dtype)


def _between_f32(dst: sp.csr_matrix) -> tuple[float, float]:
    """Interval bounds just off two stored float32 distances: float64 compares them differently from float32."""
    v = np.unique(dst.data[dst.data > 0])
    lo, hi = float(v[len(v) // 4]), float(v[3 * len(v) // 4])
    return lo + float(np.spacing(np.float32(lo))) * 0.3, hi - float(np.spacing(np.float32(hi))) * 0.3


def _pp_cases(rng):
    f32, f64 = np.float32, np.float64
    cases = {}
    for dt in (f32, f64):
        tag = np.dtype(dt).name
        cases[f"same_{tag}_interval"] = (_pair(rng, 30, same=True, dst_dtype=dt), [["interval", 2.0, 7.5]])
        cases[f"same_{tag}_interval_zeros_empty"] = (_pair(rng, 30, same=True, dst_dtype=dt, zeros=6, empty=4), [["interval", 1.5, 8.0]])
        cases[f"diff_{tag}_pct50"] = (_pair(rng, 30, same=False, dst_dtype=dt), [["percentile", 50.0]])
        cases[f"diff_{tag}_pct_zeros_empty"] = (_pair(rng, 35, same=False, dst_dtype=dt, zeros=8, empty=5), [["percentile", 62.5]])
        for q in (0.0, 100.0, 37.5):
            cases[f"ties_{tag}_pct{q:g}"] = (_pair(rng, 25, same=False, dst_dtype=dt, ties=True, zeros=3), [["percentile", q]])
        cases[f"weighted_{tag}_cosine"] = (_pair(rng, 30, same=False, dst_dtype=dt, weighted=True, zeros=5, empty=3), [["transform", "cosine"]])
        cases[f"weighted_{tag}_none"] = (_pair(rng, 30, same=False, dst_dtype=dt, weighted=True, zeros=5), [["transform", None]])
        cases[f"chain2_{tag}_pct_cosine"] = (_pair(rng, 40, same=False, dst_dtype=dt, zeros=4, empty=3), [["percentile", 80.0], ["transform", "cosine"]])
        cases[f"chain2_{tag}_interval_pct"] = (_pair(rng, 40, same=True, dst_dtype=dt, zeros=4), [["interval", 1.0, 9.0], ["percentile", 40.0]])
        cases[f"chain3_{tag}"] = (_pair(rng, 40, same=True, dst_dtype=dt, weighted=True, zeros=6, empty=2),
                                  [["interval", 0.75, 8.5], ["percentile", 70.0], ["transform", "cosine"]])
        cases[f"chain3_{tag}_none"] = (_pair(rng, 40, same=True, dst_dtype=dt, zeros=6, empty=2, ties=True),
                                       [["interval", 1.0, 3.0], ["percentile", 50.0], ["transform", None]])
        cases[f"diff_{tag}_interval_refused"] = (_pair(rng, 20, same=False, dst_dtype=dt), [["interval", 1.0, 5.0]])
    adj, dst = _pair(rng, 40, same=True, dst_dtype=f32, zeros=3)
    cases["f32_interval_between_neighbours"] = ((adj, dst), [["interval", *_between_f32(dst)]])
    adj, dst = _pair(rng, 40, same=True, dst_dtype=f64, zeros=3)
    cases["f64_interval_between_neighbours"] = ((adj, dst), [["interval", *_between_f32(dst)]])
    return cases


def _run_chain(nb, adj, dst, steps):
    adj, dst = adj.copy(), dst.copy()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for step in steps:
            if step[0] == "interval":
                post = nb.DistanceIntervalPostprocessor((step[1], step[2]))
            elif step[0] == "percentile":
                post = nb.PercentilePostprocessor(step[1])
            else:
                post = nb.TransformPostprocessor(nb.Transform.NONE if step[1] is None else nb.Transform(step[1]))
            adj, dst = post(adj, dst)
    return adj, dst


def _combine_cases(rng):
    cases = {}
    sizes = [9, 14, 7]
    perm = rng.permutation(sum(sizes))
    ixs, at = [], 0
    for s in sizes:
        ixs.extend(sorted(perm[at : at + s].tolist()))
        at += s
    for dt in (np.float32, np.float64):
        tag = np.dtype(dt).name
        blocks = [_pair(rng, s, same=False, dst_dtype=dt, zeros=2) for s in sizes]
        cases[f"interleaved_{tag}"] = (blocks, ixs)
        cases[f"contiguous_{tag}"] = (blocks, list(range(sum(sizes))))
    blocks = [_pair(rng, s, same=False, dst_dtype=np.float64, zeros=2) for s in sizes]
    cases["unsorted_within_block"] = (blocks, perm.tolist())
    return cases


def _resolve_grid():
    for coord_type, has_uns, n_neighs, radius, delaunay, percentile in itertools.product(
        (None, "grid", "generic"), (False, True), (None, 4), (None, 2.5, (1.0, 3.0)), (None, False, True), (None, 50.0)
    ):
        yield dict(coord_type=coord_type, n_neighs=n_neighs, radius=radius, delaunay=delaunay, n_rings=2 if n_neighs == 4 else None,
                   percentile=percentile, transform="cosine" if has_uns else None, set_diag=has_uns, has_spatial_uns=has_uns)


def main() -> None:
    nb, build, logged = _reference()
    rng = np.random.default_rng(20261018)
    out: dict[str, np.ndarray] = {}
    names = []
    for name, ((adj, dst), steps) in _pp_cases(rng).items():
        names.append(name)
        _put(out, f"pp/{name}/adj_in", adj)
        _put(out, f"pp/{name}/dst_in", dst)
        out[f"pp/{name}/steps"] = np.array(json.dumps(steps))
        try:
            ra, rd = _run_chain(nb, adj, dst, steps)
        except Exception as e:  # noqa: BLE001 - the reference's refusal is the expected answer
            out[f"pp/{name}/error"] = np.array(type(e).__name__)
            continue
        _put(out, f"pp/{name}/adj_out", ra)
        _put(out, f"pp/{name}/dst_out", rd)
    out["pp_cases"] = np.array(names)

    class _Blocks(nb.GraphBuilderCSR):
        def build_graph(self, coords):
            raise NotImplementedError

        def uns_params(self):
            return {}

    names = []
    for name, (blocks, ixs) in _combine_cases(rng).items():
        names.append(name)
        for b, (adj, dst) in enumerate(blocks):
            _put(out, f"combine/{name}/{b}/adj", adj)
            _put(out, f"combine/{name}/{b}/dst", dst)
        out[f"combine/{name}/ixs"] = np.asarray(ixs, dtype=np.int64)
        ra, rd = _Blocks().combine([(a.copy(), d.copy()) for a, d in blocks], ixs)
        _put(out, f"combine/{name}/adj_out", ra)
        _put(out, f"combine/{name}/dst_out", rd)
    out["combine_cases"] = np.array(names)

    records = []
    for kw in _resolve_grid():
        logged.clear()
        rec: dict = {"kwargs": kw}
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            try:
                b = build._resolve_graph_builder(**kw)
            except Exception as e:  # noqa: BLE001
                rec["error"] = [type(e).__name__, str(e)]
            else:
                rec["builder"] = type(b).__name__
                rec["uns_params"] = b.uns_params()
                rec["postprocessors"] = [[type(p).__name__, getattr(p, next(iter(p.__dataclass_fields__)))] for p in b.postprocessors()]
        rec["future_warnings"] = [str(w.message) for w in caught if issubclass(w.category, FutureWarning)]
        rec["logged"] = list(logged)
        records.append(rec)
    out["resolve"] = np.array(json.dumps(records, default=lambda v: getattr(v, "v", str(v))))

    # reference tests/graph/test_spatial_neighbors.py:82-116 and the fixtures of tests/conftest.py:207-215, 356-402
    out["known/visium_coords"] = np.array([
        [4193, 7848], [4469, 7848], [4400, 7968], [4262, 7729], [3849, 7968], [4124, 7729], [4469, 7609], [3987, 8208], [4331, 8088],
        [4262, 7968], [4124, 7968], [4124, 7489], [4537, 7968], [4469, 8088], [4331, 7848], [4056, 7848], [3849, 7729], [4262, 7489],
        [4400, 8208], [4056, 7609], [3987, 7489], [4262, 8208], [4400, 7489], [4537, 7729], [4606, 7848], [3987, 7968], [3918, 8088],
        [3918, 7848], [4193, 8088], [4056, 8088], [4193, 7609], [3987, 7729], [4331, 7609], [4124, 8208], [3780, 7848], [3918, 7609],
        [4400, 7729]], dtype=np.int64)
    out["known/visium_rings_conn_dist"] = np.array([[1, 6, 0], [2, 18, 30], [3, 36, 84]], dtype=np.int64)
    grid_rng = np.random.default_rng(42)
    out["known/squaregrid_coords"] = np.unique(grid_rng.integers(0, 10, size=(400, 2)), axis=0)
    out["known/squaregrid_rings_degree"] = np.array([[1, 4], [2, 12], [3, 24]], dtype=np.int64)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays")


if __name__ == "__main__":
    main()
