"""``squidpy_b200.gr.neighbors`` on the host: the public names, ``spatial_neighbors``' builder resolution and warnings, the
scipy post-processors and ``GraphBuilderCSR.combine`` against the unmodified reference (``tests/golden/postprocessors.npz``,
written by ``make_golden_postprocessors.py``), and custom builders through ``spatial_neighbors_from_builder``."""

from __future__ import annotations

import builtins
import json
import logging
import os
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from squidpy_b200 import _lib
from squidpy_b200._constants import Transform
from squidpy_b200.gr import neighbors as nb
from squidpy_b200.gr._build import _resolve_graph_builder

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "postprocessors.npz"))
RESOLVE = json.loads(str(GOLD["resolve"]))
REFERENCE_ALL = ["GraphMatrixT", "GraphBuilder", "GraphBuilderCSR", "GraphPostprocessor", "DistanceIntervalPostprocessor", "PercentilePostprocessor",
                 "TransformPostprocessor", "KNNBuilder", "RadiusBuilder", "DelaunayBuilder", "GridBuilder"]


def gold_csr(prefix: str) -> sp.csr_matrix:
    n = int(GOLD[f"{prefix}/n"])
    return sp.csr_matrix((GOLD[f"{prefix}/data"].copy(), GOLD[f"{prefix}/indices"].astype(np.int32), GOLD[f"{prefix}/indptr"].astype(np.int32)),
                         shape=(n, n))


def make_step(step):
    if step[0] == "interval":
        return nb.DistanceIntervalPostprocessor((step[1], step[2]))
    if step[0] == "percentile":
        return nb.PercentilePostprocessor(step[1])
    return nb.TransformPostprocessor(Transform.NONE if step[1] is None else Transform(step[1]))


def assert_same_csr(got, want: sp.csr_matrix) -> None:
    """Same stored entries (explicit zeros included), value dtype and values, bit for bit, after sort_indices()."""
    got, want = sp.csr_matrix(got, copy=True), sp.csr_matrix(want, copy=True)
    got.sort_indices()
    want.sort_indices()
    assert got.shape == want.shape
    np.testing.assert_array_equal(np.asarray(got.indptr, np.int64), np.asarray(want.indptr, np.int64))
    np.testing.assert_array_equal(np.asarray(got.indices, np.int64), np.asarray(want.indices, np.int64))
    assert got.data.dtype == want.data.dtype
    np.testing.assert_array_equal(got.data.view(np.uint8), want.data.view(np.uint8))


def test_neighbors_exports_the_reference_names_and_the_builtin_builders():
    assert nb.__all__ == REFERENCE_ALL
    for name in REFERENCE_ALL:
        assert hasattr(nb, name)
    assert nb.KNNBuilder is sq.gr.KNNBuilder
    assert nb.RadiusBuilder is sq.gr.RadiusBuilder
    assert nb.DelaunayBuilder is sq.gr.DelaunayBuilder
    assert nb.GridBuilder is sq.gr.GridBuilder
    assert sq.gr.spatial_neighbors in (getattr(sq.gr, n) for n in sq.gr.__all__)
    for cls in (nb.KNNBuilder, nb.RadiusBuilder, nb.DelaunayBuilder, nb.GridBuilder):
        assert issubclass(cls, nb.GraphBuilderCSR) and issubclass(cls, nb.GraphBuilder)
    for cls in (nb.DistanceIntervalPostprocessor, nb.PercentilePostprocessor, nb.TransformPostprocessor):
        with pytest.raises(Exception):  # frozen dataclasses
            setattr(cls(1.0) if cls is not nb.DistanceIntervalPostprocessor else cls((0.0, 1.0)), "x", 1)


@pytest.mark.parametrize("name", [str(n) for n in GOLD["pp_cases"]])
def test_host_postprocessors_equal_reference(name):
    adj, dst = gold_csr(f"pp/{name}/adj_in"), gold_csr(f"pp/{name}/dst_in")
    steps = json.loads(str(GOLD[f"pp/{name}/steps"]))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", sp.SparseEfficiencyWarning)
        if f"pp/{name}/error" in GOLD:
            with pytest.raises(getattr(builtins, str(GOLD[f"pp/{name}/error"]))):
                for step in steps:
                    adj, dst = make_step(step)(adj, dst)
            return
        for step in steps:
            adj, dst = make_step(step)(adj, dst)
    assert_same_csr(adj, gold_csr(f"pp/{name}/adj_out"))
    assert_same_csr(dst, gold_csr(f"pp/{name}/dst_out"))


class _Blocks(nb.GraphBuilderCSR):
    def build_graph(self, coords):
        raise NotImplementedError

    def uns_params(self):
        return {}


def combine_blocks(name: str):
    blocks, b = [], 0
    while f"combine/{name}/{b}/adj/n" in GOLD:
        blocks.append((gold_csr(f"combine/{name}/{b}/adj"), gold_csr(f"combine/{name}/{b}/dst")))
        b += 1
    return blocks, GOLD[f"combine/{name}/ixs"].tolist()


@pytest.mark.parametrize("name", [str(n) for n in GOLD["combine_cases"]])
def test_host_combine_equals_reference(name):
    blocks, ixs = combine_blocks(name)
    adj, dst = _Blocks().combine(blocks, ixs)
    assert_same_csr(adj, gold_csr(f"combine/{name}/adj_out"))
    assert_same_csr(dst, gold_csr(f"combine/{name}/dst_out"))


def test_base_class_combine_raises_the_reference_error():
    class Plain(nb.GraphBuilder):
        def build_graph(self, coords):
            return None, None

        def uns_params(self):
            return {}

    with pytest.raises(NotImplementedError, match="Using `library_key` with this graph builder is not implemented yet."):
        Plain().combine([], [])


def _resolve_kwargs(kw: dict) -> dict:
    kw = dict(kw)
    if isinstance(kw["radius"], list):
        kw["radius"] = tuple(kw["radius"])
    return kw


def test_resolution_matches_reference(caplog):
    for rec in RESOLVE:
        kw = _resolve_kwargs(rec["kwargs"])
        caplog.clear()
        with warnings.catch_warnings(record=True) as caught, caplog.at_level(logging.WARNING, logger="squidpy_b200"):
            warnings.simplefilter("always")
            try:
                b = _resolve_graph_builder(**kw)
            except NotImplementedError:
                # GridBuilder(delaunay=True) needs Qhull's Delaunay triangulation and is refused here
                assert rec.get("builder") == "GridBuilder" and kw["delaunay"], rec
                continue
            except Exception as e:  # noqa: BLE001
                assert "error" in rec, (rec, e)
                assert [type(e).__name__, str(e)] == rec["error"]
                continue
        assert "error" not in rec, rec
        assert type(b).__name__ == rec["builder"]
        assert json.loads(json.dumps(b.uns_params(), default=lambda v: getattr(v, "v", str(v)))) == rec["uns_params"]
        got = [[type(p).__name__, getattr(p, next(iter(p.__dataclass_fields__)))] for p in b.postprocessors()]
        assert json.loads(json.dumps(got, default=lambda v: getattr(v, "v", str(v)))) == rec["postprocessors"]
        assert [str(w.message) for w in caught if issubclass(w.category, FutureWarning)] == rec["future_warnings"]
        assert [r.getMessage() for r in caplog.records] == rec["logged"]


def test_spatial_neighbors_raises_the_deprecation_warning_and_refuses_grid_percentile():
    co = np.random.default_rng(0).uniform(0, 100, (40, 2))
    adata = sq.AnnDataLite(obsm={"spatial": co}, shape=(40, 0))
    with pytest.warns(FutureWarning, match="Calling `spatial_neighbors` is deprecated and will be removed in squidpy v1.9.0"):
        with pytest.raises(ValueError, match="`percentile` is not supported for grid coordinates"):
            sq.gr.spatial_neighbors(adata, coord_type="grid", percentile=50.0)
    with pytest.warns(FutureWarning):
        with pytest.raises(NotImplementedError):
            sq.gr.spatial_neighbors(adata, coord_type="grid", delaunay=True)


class HostKNN(nb.GraphBuilderCSR):
    """A caller's builder: a kNN graph in numpy / scipy, post-processed by the public classes."""

    def __init__(self, k=4, percentile=None, transform=None):
        steps = [] if percentile is None else [nb.PercentilePostprocessor(percentile)]
        super().__init__(transform=transform, percentile=percentile,
                         postprocessors=[*steps, nb.TransformPostprocessor(Transform.NONE if transform is None else Transform(transform))])
        self.k = k
        self.calls = 0

    def build_graph(self, coords):
        self.calls += 1
        co = np.asarray(coords, dtype=np.float64)
        d = np.linalg.norm(co[:, None] - co[None], axis=-1)
        np.fill_diagonal(d, np.inf)
        nn = np.sort(np.argsort(d, axis=1, kind="stable")[:, : self.k], axis=1)
        n = co.shape[0]
        rows = np.repeat(np.arange(n), self.k)
        adj = sp.csr_matrix((np.ones(n * self.k, np.float32), (rows, nn.ravel())), shape=(n, n))
        dst = sp.csr_matrix((d[rows, nn.ravel()], (rows, nn.ravel())), shape=(n, n))
        return adj, dst

    def uns_params(self):
        return {"coord_type": "generic", "n_neighbors": self.k, "transform": self.transform.v}


def test_custom_builder_through_spatial_neighbors_from_builder():
    rng = np.random.default_rng(5)
    co = rng.uniform(0, 100, (60, 2))
    codes = rng.integers(0, 3, 60)
    obs = pd.DataFrame({"lib": pd.Categorical.from_codes(codes, ["a", "b", "c"])})
    builder = HostKNN(k=4, percentile=75.0, transform="cosine")
    adata = sq.AnnDataLite(obs=obs, obsm={"spatial": co}, shape=(60, 0))
    sq.gr.spatial_neighbors_from_builder(adata, builder)
    want = builder.build(co)
    assert_same_csr(adata.obsp["spatial_connectivities"], sp.csr_matrix(want[0]))
    assert adata.uns["spatial_neighbors"]["params"] == builder.uns_params()

    builder.calls = 0
    res = sq.gr.spatial_neighbors_from_builder(adata, builder, library_key="lib", copy=True)
    assert builder.calls == 3
    mats, ixs = [], []
    for code in range(3):
        idx = np.where(codes == code)[0]
        mats.append(builder.build(co[idx]))
        ixs.extend(idx.tolist())
    adj, dst = builder.combine(mats, ixs)
    assert_same_csr(res.connectivities, sp.csr_matrix(adj))
    assert_same_csr(res.distances, sp.csr_matrix(dst))

    with pytest.raises(TypeError, match="Expected a graph builder"):
        sq.gr.spatial_neighbors_from_builder(adata, object())

    class NoCombine(nb.GraphBuilder):
        def build_graph(self, coords):
            return HostKNN().build_graph(coords)

        def uns_params(self):
            return {}

    with pytest.raises(NotImplementedError, match="Using `library_key`"):
        sq.gr.spatial_neighbors_from_builder(adata, NoCombine(), library_key="lib")


def test_builtin_builders_declare_the_reference_postprocessors():
    assert nb.KNNBuilder(percentile=30.0, transform="cosine").postprocessors() == [nb.PercentilePostprocessor(30.0),
                                                                                  nb.TransformPostprocessor(Transform.COSINE)]
    assert nb.RadiusBuilder(radius=(4.0, 1.0)).postprocessors() == [nb.DistanceIntervalPostprocessor((1.0, 4.0)),
                                                                   nb.TransformPostprocessor(Transform.NONE)]
    assert nb.RadiusBuilder(radius=2.0, percentile=5.0).postprocessors() == [nb.PercentilePostprocessor(5.0), nb.TransformPostprocessor(Transform.NONE)]
    assert nb.DelaunayBuilder(radius=3).postprocessors() == [nb.DistanceIntervalPostprocessor((0.0, 3.0)), nb.TransformPostprocessor(Transform.NONE)]
    assert nb.GridBuilder(transform="spectral").postprocessors() == [nb.TransformPostprocessor(Transform.SPECTRAL)]


def test_abi_version_and_symbols_are_declared():
    assert "sqb_graph_postprocess" in _lib.EXPORTED_SYMBOLS and "sqb_graph_combine" in _lib.EXPORTED_SYMBOLS
    assert _lib.ABI_VERSION == 18
    lib = _lib.load()
    assert lib.sqb_abi_version() == 18
    assert hasattr(lib, "sqb_graph_postprocess") and hasattr(lib, "sqb_graph_combine")
