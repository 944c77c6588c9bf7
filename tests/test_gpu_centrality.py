"""sqb_centrality_scores on the GPU against the restatement ``tests/centrality_ref.py``, bit for bit: every golden case,
deep BFS (a 200 000-node path, a 2 000 x 500 lattice), 1M-spot hex grids with 20 and 150 clusters, an empty graph, and
device graphs (torch ``sparse_csr`` / ``sparse_csc``, int64 indices) against the same graph from the host."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from squidpy_b200.gr._nhood import centrality_counts
from tests import centrality_ref
from tests.golden.make_golden_centrality import SCORES, make_adata
from tests.test_centrality_host import GOLDEN, N_CASES, golden_case
from tools import synth

pytestmark = pytest.mark.gpu


def _check(graph, codes, n_cls, ref=None):
    ref = ref or centrality_ref.counts(graph, codes, n_cls)
    got = centrality_counts(graph, codes, n_cls, 7)
    np.testing.assert_array_equal(got.reach1, ref.reach1)
    np.testing.assert_array_equal(got.dist, ref.dist)
    np.testing.assert_array_equal(got.cc, ref.cc)
    assert got.levels == ref.levels
    return got


@pytest.mark.parametrize("case", range(N_CASES))
def test_golden_case_kernels_and_frames(case):
    g = np.load(GOLDEN)
    graph, codes, n_cls = golden_case(g, case)
    _check(graph, codes, n_cls)
    for j, score in enumerate(SCORES):
        df = sq.gr.centrality_scores(make_adata(graph, codes, n_cls), "cluster", score=score, copy=True)
        np.testing.assert_array_equal(df.to_numpy(), g[f"c{case}_s{j}_values"])
        assert list(df.columns) == list(g[f"c{case}_s{j}_cols"])


def test_single_measures_match_full_run():
    graph, codes, n_cls = golden_case(np.load(GOLDEN), 0)
    full = centrality_counts(graph, codes, n_cls, 7)
    deg = centrality_counts(graph, codes, n_cls, 1)
    assert deg.dist is None and deg.cc is None and deg.levels == -1
    np.testing.assert_array_equal(deg.reach1, full.reach1)
    np.testing.assert_array_equal(centrality_counts(graph, codes, n_cls, 2).dist, full.dist)
    np.testing.assert_array_equal(centrality_counts(graph, codes, n_cls, 4).cc, full.cc)


def _path(n):
    i = np.arange(n - 1)
    return sp.csr_matrix((np.ones(n - 1, np.float32), (i, i + 1)), shape=(n, n))  # one direction only


def test_path_graph_200k():
    n = 200_000
    codes = np.full(n, -1)
    codes[0], codes[n // 2], codes[n - 1] = 0, 1, 0
    got = _check(_path(n), codes, 2)
    assert got.levels == n // 2  # from the middle node to node 0


def test_lattice_2000x500():
    rows, cols = 2000, 500
    idx = np.arange(rows * cols).reshape(rows, cols)
    r = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
    c = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    g = sp.csr_matrix((np.ones(r.size), (r, c)), shape=(rows * cols,) * 2)
    codes = np.full(rows * cols, -1)
    codes[idx[0, 0]], codes[idx[-1, -1]], codes[idx[1000, 250]] = 0, 1, 2
    got = _check(g, codes, 3)
    assert got.levels == rows - 1 + cols - 1


@pytest.mark.parametrize("n_cls,stripes", [(20, True), (150, False)])
def test_hex_1m(n_cls, stripes):
    g = synth.hex_graph(1000, 1000)
    if stripes:  # spatially coherent clusters: a deep BFS
        codes = (np.arange(1_000_000) % 1000) * n_cls // 1000
    else:
        codes = np.random.default_rng(n_cls).integers(0, n_cls, 1_000_000)
    got = _check(g, codes, n_cls)
    assert got.levels > (900 if stripes else 2)


def test_empty_graph():
    n = 50
    g = sp.csr_matrix((n, n), dtype=np.float64)
    codes = np.arange(n) % 3
    got = _check(g, codes, 4)
    assert got.levels == 0 and (got.reach1 == 0).all() and (got.cc == 0).all()
    df = sq.gr.centrality_scores(make_adata(g, codes, 4), "cluster", copy=True)
    assert (df["degree_centrality"] == 0).all() and (df["closeness_centrality"].iloc[:3] == 0).all()
    assert np.isnan(df["closeness_centrality"].iloc[3])


def _torch_graph(m, layout, index_dtype):
    import torch

    if layout == "csr":
        m = m.tocsr()
        t = torch.sparse_csr_tensor(torch.from_numpy(m.indptr.astype(index_dtype)), torch.from_numpy(m.indices.astype(index_dtype)),
                                    torch.from_numpy(m.data), size=m.shape)
    else:
        m = m.tocsc()
        t = torch.sparse_csc_tensor(torch.from_numpy(m.indptr.astype(index_dtype)), torch.from_numpy(m.indices.astype(index_dtype)),
                                    torch.from_numpy(m.data), size=m.shape)
    return t.cuda()


@pytest.mark.parametrize("layout", ["csr", "csc"])
@pytest.mark.parametrize("index_dtype", [np.int32, np.int64])
@pytest.mark.parametrize("case", [0, 2, 3, 4, 6, 7, 13, 14, 20])  # float32, float64, int64, int32 and bool values
def test_device_graph_equals_host(layout, index_dtype, case):
    graph, codes, n_cls = golden_case(np.load(GOLDEN), case)
    host = sq.gr.centrality_scores(make_adata(graph, codes, n_cls), "cluster", copy=True)
    dev = sq.gr.centrality_scores(make_adata(_torch_graph(graph, layout, index_dtype), codes, n_cls), "cluster", copy=True)
    assert dev.equals(host)


def test_device_graph_cancellation_and_bad_index():
    import torch

    g = golden_case(np.load(GOLDEN), 4)[0]  # handmade float64: (3, 4) cancels
    codes = np.array([0, 0, 1, 1, 2, 2, 2, 0, 1, -1, 2])
    d = centrality_counts(_torch_graph(g, "csr", np.int64), codes, 3, 7)
    h = centrality_counts(g, codes, 3, 7)
    np.testing.assert_array_equal(d.dist, h.dist)
    np.testing.assert_array_equal(d.cc, h.cc)
    bad = torch.sparse_csr_tensor(torch.tensor([0, 1, 1]), torch.tensor([5]), torch.tensor([1.0]), size=(2, 2)).cuda()
    with pytest.raises(ValueError, match="out of range"):
        centrality_counts(bad, np.array([0, 1]), 2, 7)
