"""centrality_scores checked without a GPU: the restatement ``tests/centrality_ref.py`` against scipy's ``A + Aᵀ`` and
networkx's group measures, and the public ``centrality_scores`` (with the device call replaced by that restatement) against
the unmodified reference's golden output, errors included."""

from __future__ import annotations

import os

import networkx as nx
import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from squidpy_b200._constants import Centrality, Key
from squidpy_b200.gr import _nhood
from tests import centrality_ref
from tests.golden.make_golden_centrality import SCORES, make_adata

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "centrality.npz")
N_CASES = 23
N_ERRORS = 6


def golden_case(g, i):
    fmt = str(g[f"c{i}_format"])
    n = g[f"c{i}_codes"].size
    graph = (sp.csr_matrix if fmt == "csr" else sp.csc_matrix)((g[f"c{i}_data"], g[f"c{i}_indices"], g[f"c{i}_indptr"]), shape=(n, n))
    return graph, g[f"c{i}_codes"], int(g[f"c{i}_ncls"])


def test_golden_case_count():
    g = np.load(GOLDEN)
    assert sum(k.endswith("_name") and k.startswith("c") for k in g.files) == N_CASES
    assert sum(k.endswith("_name") and k.startswith("e") for k in g.files) == N_ERRORS


@pytest.mark.parametrize("case", range(N_CASES))
def test_canonical_graph_is_scipy_sum(case):
    """The sort-and-segment restatement == the reference's ``A + Aᵀ``, ``setdiag(0)``, ``eliminate_zeros``."""
    graph, _, _ = golden_case(np.load(GOLDEN), case)
    adj = sp.csr_matrix(graph)
    adj = (adj + adj.T).tocsr()
    adj.setdiag(0)
    adj.eliminate_zeros()
    adj.sort_indices()
    got = centrality_ref.canonical(graph)
    np.testing.assert_array_equal(got.indptr, adj.indptr)
    np.testing.assert_array_equal(got.indices, adj.indices)


def test_canonical_cancellations():
    """The golden's hand-made graphs drop the pair (3, 4) by cancellation in every dtype but bool, the explicit zero (2, 3)
    everywhere, and the self loop (0, 0)."""
    g = np.load(GOLDEN)
    names = [str(g[f"c{i}_name"]) for i in range(N_CASES)]
    for i, name in enumerate(names):
        if not name.startswith("handmade"):
            continue
        c = centrality_ref.canonical(golden_case(g, i)[0])
        assert c[3, 4] == (name == "handmade_bool"), name
        assert not c[2, 3] and not c[0, 0], name


@pytest.mark.parametrize("case", range(N_CASES))
def test_restatement_matches_networkx(case):
    graph, codes, n_cls = golden_case(np.load(GOLDEN), case)
    ref = centrality_ref.counts(graph, codes, n_cls)
    G = nx.Graph()
    G.add_nodes_from(range(codes.size))
    c = sp.triu(centrality_ref.canonical(graph), k=1).tocoo()
    G.add_edges_from(zip(c.row.tolist(), c.col.tolist()))
    n = codes.size
    cc = nx.clustering(G)
    np.testing.assert_array_equal(ref.cc, np.array([cc[v] for v in range(n)], dtype=np.float64))
    for k in range(n_cls):
        idx = np.flatnonzero(codes == k).tolist()
        if idx and len(idx) < n:
            assert ref.reach1[k] / (n - len(idx)) == nx.group_degree_centrality(G, idx)
            d = ref.dist[k]
            assert ((n - len(idx)) / d if d else 0.0) == nx.group_closeness_centrality(G, idx)


@pytest.fixture()
def host_kernel(monkeypatch):
    """``centrality_counts`` replaced by the restatement: the measures the device would be asked for are recorded."""
    calls = []

    def fake(conn, codes, n_cls, measures, *, device=None):
        calls.append(measures)
        r = centrality_ref.counts(conn, codes, n_cls)
        return _nhood.CentralityCounts(r.reach1 if measures & 1 else None, r.dist if measures & 2 else None,
                                       r.cc if measures & 4 else None, r.levels if measures & 2 else -1)

    monkeypatch.setattr(_nhood, "centrality_counts", fake)
    return calls


@pytest.mark.parametrize("case", range(N_CASES))
def test_reproduces_reference_golden(host_kernel, case):
    g = np.load(GOLDEN)
    graph, codes, n_cls = golden_case(g, case)
    for j, score in enumerate(SCORES):
        df = sq.gr.centrality_scores(make_adata(graph, codes, n_cls), "cluster", score=score, copy=True)
        assert list(df.columns) == list(g[f"c{case}_s{j}_cols"])
        assert [str(t) for t in df.dtypes] == list(g[f"c{case}_s{j}_dtypes"])
        assert list(df.index) == [f"c{k}" for k in range(n_cls)]
        np.testing.assert_array_equal(df.to_numpy(), g[f"c{case}_s{j}_values"])
    assert host_kernel == [7, 1, 4, 2]


def test_undefined_measures_are_nan(host_kernel):
    g = np.load(GOLDEN)
    names = [str(g[f"c{i}_name"]) for i in range(N_CASES)]
    one = g[f"c{names.index('one_category')}_s0_values"]
    assert np.isnan(one[0, 0]) and one[0, 2] == 0.0  # degree of the group of every node; closeness with nothing outside
    unused = g[f"c{names.index('hex_nan_unused')}_s0_values"]
    assert np.isnan(unused[3, 2]) and np.isnan(unused[5, 2])  # closeness of the unused categories
    assert unused[3, 0] == 0.0 and unused[3, 1] == 0.0


def test_stores_in_uns_and_accepts_enum(host_kernel):
    g = np.load(GOLDEN)
    graph, codes, n_cls = golden_case(g, 0)
    a = make_adata(graph, codes, n_cls)
    assert sq.gr.centrality_scores(a, "cluster", n_jobs=4, backend="threading", show_progress_bar=True) is None
    stored = a.uns[Key.uns.centrality_scores("cluster")]
    assert isinstance(stored, pd.DataFrame)
    np.testing.assert_array_equal(stored.to_numpy(), g["c0_s0_values"])
    df = sq.gr.centrality_scores(a, "cluster", score=Centrality.CLOSENESS, copy=True)
    np.testing.assert_array_equal(df.to_numpy(), g["c0_s3_values"])


@pytest.mark.parametrize("err", range(N_ERRORS))
def test_reference_errors(host_kernel, err):
    from tests.golden.make_golden_centrality import _labels, error_cases
    from tools import synth

    g = np.load(GOLDEN)
    name, factory, kw = error_cases(synth.hex_graph(4, 4), _labels(16, 3, 9))[err]
    assert name == str(g[f"e{err}_name"])
    with pytest.raises(Exception) as info:
        sq.gr.centrality_scores(factory(), copy=True, **kw)
    assert type(info.value).__name__ == str(g[f"e{err}_type"])
    assert str(info.value) == str(g[f"e{err}_msg"])
    assert host_kernel == []


def test_unsupported_host_value_dtype():
    a = sp.csr_matrix(np.eye(3, dtype=np.complex64))
    with pytest.raises(TypeError, match="complex64"):
        _nhood.centrality_counts(a, np.zeros(3, dtype=np.int32), 1, 7)
