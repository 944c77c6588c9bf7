"""calculate_niche without a GPU: the numpy restatement of the embeddings against the reference's golden, argument
validation, warnings, postprocessing and AnnDataLite's row subsets."""

from __future__ import annotations

import json
import logging
import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

from squidpy_b200._adata import AnnDataLite
from squidpy_b200.gr import _niche
from tests import niche_ref
from tests import niche_scanpy_standin as standin
from tests.golden.make_golden_niche import build_call, cases, error_cases, graphs, make_adata, warning_cases

GOLD = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "niche.npz"), allow_pickle=False))
CASES = cases()
GRAPHS = graphs()


def golden_calls(i):
    return [(str(GOLD[f"c{i}_k{j}_name"]), GOLD[f"c{i}_k{j}_X"], json.loads(str(GOLD[f"c{i}_k{j}_info"])))
            for j in range(int(GOLD[f"c{i}_ncalls"]))]


def embedding_of(case, adata, kw):
    """The restatement's embedding for a single-library case, as handed to the first scanpy call."""
    _, fn, _, _ = case
    A = adata.obsp["spatial_connectivities"]
    if fn == "calculate_niche":
        fn = kw["flavor"]
        kw = {**kw, "distance": kw.get("distance", 3 if fn == "cellcharter" else 1)}
    if fn == "neighborhood":
        col = adata.obs[kw["groups"]]
        return niche_ref.profile(A, col.cat.codes.to_numpy(), len(col.cat.categories), kw.get("distance", 1), kw.get("n_hop_weights"),
                                 kw.get("abs_nhood", False))
    if fn == "utag":
        return niche_ref.utag(A, adata.X)
    return niche_ref.cellcharter(A, adata.X, kw.get("distance", 3), kw.get("aggregation", "mean"))[0]


@pytest.mark.parametrize("i", [i for i, c in enumerate(CASES) if "library_key" not in c[3] and "use_rep" not in c[3]],
                         ids=lambda i: CASES[i][0])
def test_restatement_matches_reference(i):
    case = CASES[i]
    adata, kw = build_call(case, GRAPHS)
    got = embedding_of(case, adata, kw)
    _, X, info = golden_calls(i)[0]
    assert got.dtype == np.dtype(info["dtype"])
    if case[1] == "cellcharter" or kw.get("flavor") == "cellcharter":
        m = adata.n_vars
        np.testing.assert_array_equal(got[:, : 2 * m], X[:, : 2 * m])  # X and hop 1: bit for bit
        np.testing.assert_allclose(got[:, 2 * m:], X[:, 2 * m:], rtol=1e-12, atol=1e-300)
    elif "weighted" in case[0] and case[1] == "neighborhood":
        np.testing.assert_allclose(got, X, rtol=1e-5)
    else:
        np.testing.assert_array_equal(got, X)


def test_hop_sets_compare_path_weights():
    # 3 x 3 king's-move lattice: a cell's path weight back to itself or to a neighbour after two hops exceeds its visited
    # value, so hop 2 of every cell holds the cell and all of its 1-hop neighbours
    r, c = np.divmod(np.arange(9), 3)
    A = sp.csr_matrix(((np.abs(r[:, None] - r) <= 1) & (np.abs(c[:, None] - c) <= 1) & ~np.eye(9, dtype=bool)).astype(np.float32))
    H2 = niche_ref.hops(A, 2)[1].toarray()
    assert H2.diagonal().all() and H2[A.toarray() > 0].all()


def test_pairwise_degree_is_numpys_reduction():
    rng = np.random.default_rng(0)
    for n in (1, 5, 8, 9, 17, 128, 129, 300):
        row = (rng.random(n) * 3).astype(np.float32)
        H = sp.csr_matrix((row, np.arange(n), [0, n]), shape=(1, 400))
        expect = row[0] + np.add.reduce(row[1:]) if n > 1 else row[0]
        assert np.asarray(H.sum(axis=1))[0, 0] == np.float32(expect)


@pytest.mark.parametrize("j", range(len(error_cases())), ids=[e[0] for e in error_cases()])
def test_errors_match_reference(j):
    name, kw = error_cases()[j]
    standin.install()
    adata = make_adata(GRAPHS["hex"], sparse_x=not name.startswith("cc_dense"))
    exc = {"ValueError": ValueError, "TypeError": TypeError, "KeyError": KeyError, "AttributeError": AttributeError}[str(GOLD[f"e{j}_type"])]
    with pytest.warns(FutureWarning, match="Calling `calculate_niche` is deprecated"):
        with pytest.raises(exc) as info:
            _niche.calculate_niche(adata, **kw)
    assert str(info.value) == str(GOLD[f"e{j}_msg"]) or (exc is KeyError and repr(str(GOLD[f"e{j}_msg"])) == str(info.value))


@pytest.mark.parametrize("j", range(len(warning_cases())), ids=[w[0] for w in warning_cases()])
def test_unused_argument_warnings_match_reference(j, caplog):
    name, kw = warning_cases()[j]
    kw = dict(kw)
    flavor = kw.pop("flavor")
    if flavor == "cellcharter":
        kw.setdefault("aggregation", "mean")
    args = dict(library_key=None, table_key=None, groups=None, n_neighbors=None, resolutions=None, min_niche_size=None, scale=True,
                abs_nhood=False, distance=3 if flavor == "cellcharter" else 1, n_hop_weights=None, aggregation=None, n_components=None,
                random_state=42, spatial_connectivities_key="spatial_connectivities", latent_connectivities_key="connectivities",
                layer_ratio=1.0, n_iterations=-1, use_weights=True, use_rep=None, inplace=True)
    args.update(kw)
    with caplog.at_level(logging.WARNING, logger="squidpy_b200"):
        _niche._validate_niche_args(make_adata(GRAPHS["hex"]), flavor, **args)
    got = [f"WARNING:{r.getMessage()}" for r in caplog.records if r.levelno == logging.WARNING]
    assert got == [str(s) for s in GOLD[f"w{j}_log"] if "not used" in str(s)]


def test_spatialleiden_not_provided():
    with pytest.raises(NotImplementedError, match="spatialleiden"):
        _niche.calculate_niche_spatialleiden(make_adata(GRAPHS["hex"]), 0.5)
    with pytest.warns(FutureWarning), pytest.raises(NotImplementedError, match="spatialleiden"):
        _niche.calculate_niche(make_adata(GRAPHS["hex"]), "spatialleiden")


def test_leiden_flavours_need_scanpy(monkeypatch):
    import sys

    monkeypatch.setitem(sys.modules, "scanpy", None)  # import scanpy -> ImportError
    adata = make_adata(GRAPHS["hex"])
    with pytest.raises(ImportError, match="scanpy"):
        _niche.calculate_niche_neighborhood(adata, "cell_type", 0.5)
    with pytest.raises(ImportError, match="scanpy"):
        _niche.calculate_niche_utag(adata, 0.5)
    with pytest.raises(ImportError, match="scanpy"):
        _niche.calculate_niche_cellcharter(adata)


def test_postprocess():
    obs = pd.DataFrame({"n": pd.Categorical([0, 0, 1, 1, 1, 2])}, index=list("abcdef"))
    a = AnnDataLite(obs=obs, shape=(6, 0))
    mask = pd.Series([True, False, True, True, True, True, False], index=list("abcdefz"))
    _niche._postprocess_niche_results(a, ["n"], mask=mask, min_niche_size=2, prefix="lib=x_")
    # "0" keeps one cell once "b" is masked, below min_niche_size like "2"
    assert list(a.obs["n"]) == ["lib=x_not_a_niche", "lib=x_not_a_niche", "lib=x_1", "lib=x_1", "lib=x_1", "lib=x_not_a_niche"]
    b = AnnDataLite(obs=pd.DataFrame({"n": pd.Categorical([0, 1])}), shape=(2, 0))
    _niche._postprocess_niche_results(b, ["n"])
    assert b.obs["n"].dtype.name == "category"


def test_anndatalite_obs_subset():
    A = sp.random(6, 6, density=0.5, format="csr", random_state=0)
    a = AnnDataLite(X=np.arange(12.0).reshape(6, 2), obs=pd.DataFrame({"k": list("xyzxyz")}, index=list("abcdef")),
                    obsm={"e": np.arange(6.0)[:, None]}, obsp={"g": A}, layers={"l": np.ones((6, 2))})
    for sub in (a[pd.Index(["f", "b"])], a[["f", "b"], :], a[np.array([5, 1])], a[np.array([False, True, False, False, False, True])][[1, 0]]):
        assert list(sub.obs.index) == ["f", "b"]
        np.testing.assert_array_equal(sub.X, a.X[[5, 1]])
        np.testing.assert_array_equal(sub.obsm["e"][:, 0], [5.0, 1.0])
        np.testing.assert_array_equal(sub.obsp["g"].toarray(), A.toarray()[np.ix_([5, 1], [5, 1])])
        assert sub.layers["l"].shape == (2, 2) and sub.shape == (2, 2)
    v = a[:, [0]]  # a variable subset keeps its behaviour
    assert v.shape == (6, 1) and v.obsp["g"] is a.obsp["g"]


def test_boolean_graphs_refused():
    # scipy's A^k of a boolean graph is reachability and its hop comparison True > True is False: path sums differ
    A = GRAPHS["hex"].astype(bool)
    codes = np.zeros(A.shape[0], dtype=np.int32)
    with pytest.raises(TypeError, match="Boolean connectivity graphs"):
        _niche.niche_profile(A, codes, 1, 2)
    with pytest.raises(TypeError, match="Boolean connectivity graphs"):
        _niche.niche_aggregate(A, make_adata(GRAPHS["hex"]).X, "mean", 2)


class _RowEmbedder:
    def embed(self, adata):
        return adata.obsm["pos"]


class _RowClusterer:
    def cluster(self, adata, embedding):
        adata.obs["n"] = pd.Categorical(embedding[:, 0].astype(int).astype(str))
        return ["n"]


def test_library_rows_by_position_with_integer_obs_names():
    # obs names 100, 99, ... are integers but not positions: every library still runs on its own rows
    n = 9
    obs = pd.DataFrame({"lib": pd.Categorical(list("abcabcabc"))}, index=np.arange(100, 100 - n, -1))
    a = AnnDataLite(obs=obs, obsm={"pos": np.arange(n, dtype=float)[:, None]}, obsp={"g": sp.identity(n, format="csr")}, shape=(n, 0))
    _niche._calculate_niche_custom(a, _RowEmbedder(), _RowClusterer(), library_key="lib")
    assert list(a.obs["n"]) == [f"lib={lib}_{i}" for i, lib in enumerate("abcabcabc")]


def test_anndatalite_obs_subset_torch_and_raw():
    import torch

    A = sp.random(6, 6, density=0.5, format="csr", random_state=1)
    t = torch.sparse_csr_tensor(torch.from_numpy(A.indptr.astype(np.int64)), torch.from_numpy(A.indices.astype(np.int64)),
                                torch.from_numpy(A.data), size=A.shape)
    raw = AnnDataLite(X=np.arange(6.0)[:, None], obs=pd.DataFrame(index=list("abcdef")))
    a = AnnDataLite(X=torch.arange(12.0).reshape(6, 2), obs=pd.DataFrame(index=list("abcdef")), obsp={"g": t}, raw=raw)
    sub = a[["e", "a", "c"]].copy()
    assert sub.obsp["g"].layout == torch.sparse_csr
    np.testing.assert_array_equal(sub.obsp["g"].to_dense().numpy(), A.toarray()[np.ix_([4, 0, 2], [4, 0, 2])])
    np.testing.assert_array_equal(sub.X.numpy(), np.arange(12.0).reshape(6, 2)[[4, 0, 2]])
    np.testing.assert_array_equal(sub.raw.X[:, 0], [4.0, 0.0, 2.0])
