"""interaction_matrix through the C ABI against the oracle (pinned to the reference kernel in test_oracle_vs_reference.py)
and against the reference's own known answers (tests/graph/test_nhood.py:153-173)."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from oracle import ref
from tools import synth

pytestmark = pytest.mark.gpu


def _adata(g, codes, n_cats):
    cat = pd.Categorical.from_codes(codes, [f"c{i}" for i in range(n_cats)])
    return synth.make_adata(np.zeros((g.shape[0], 2)), g, pd.Series(cat), cluster_key="cat")


def test_known_answers_of_the_reference():
    g = sp.csr_matrix(np.array([[0, 1, 1, 0, 0], [0, 0, 0, 0, 1], [1, 2, 0, 0, 0], [0, 1, 0, 0, 1], [0, 0, 1, 2, 0]]))
    ad = _adata(g, [0, 0, 0, 1, 1], 2)
    w = sq.gr.interaction_matrix(ad, "cat", weights=True, copy=True)
    u = sq.gr.interaction_matrix(ad, "cat", weights=False, copy=True)
    np.testing.assert_array_equal(w, [[5, 1], [2, 3]])
    np.testing.assert_array_equal(u, [[4, 1], [2, 2]])
    assert w.dtype == np.int64 and u.dtype == np.int64  # integer graph -> int output (_nhood.py:398)
    ad = _adata(g, [-1, 0, 0, 1, 1], 2)  # NaN label on observation 0
    np.testing.assert_array_equal(sq.gr.interaction_matrix(ad, "cat", weights=True, copy=True), [[2, 1], [2, 3]])
    np.testing.assert_array_equal(sq.gr.interaction_matrix(ad, "cat", weights=False, copy=True), [[1, 1], [2, 2]])
    sq.gr.interaction_matrix(ad, "cat")
    np.testing.assert_array_equal(ad.uns["cat_interactions"], [[1, 1], [2, 2]])
    with pytest.raises(RuntimeError, match="none remain"):
        sq.gr.interaction_matrix(_adata(g, [-1] * 5, 2), "cat", copy=True)


@pytest.mark.parametrize("n_cats", [2, 9, 40, 120])
@pytest.mark.parametrize("weights", [False, True])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_random_graphs_vs_oracle(n_cats, weights, dtype):
    rng = np.random.default_rng(n_cats)
    n = 6000
    g = sp.random(n, n, density=0.002, format="csr", random_state=3, dtype=dtype)
    codes = rng.integers(-1, n_cats, n)  # some NaN labels
    exp = ref.interaction_matrix(g, codes, n_cats, weights=weights)
    got = sq.gr.interaction_matrix(_adata(g, codes, n_cats), "cat", weights=weights, copy=True)
    assert got.dtype == np.float64
    assert got.tobytes() == exp.tobytes()  # float64 sums in the reference's order: the same bits
    expn = ref.interaction_matrix(g, codes, n_cats, weights=weights, normalized=True)
    gotn = sq.gr.interaction_matrix(_adata(g, codes, n_cats), "cat", weights=weights, normalized=True, copy=True)
    assert gotn.dtype == expn.dtype and np.array_equal(gotn, expn, equal_nan=True) and (np.signbit(gotn) == np.signbit(expn)).all()


def test_equals_the_nhood_count_on_a_lattice():
    g = synth.hex_graph(101, 97)
    codes = np.random.default_rng(0).integers(0, 13, g.shape[0])
    got = sq.gr.interaction_matrix(_adata(g, codes, 13), "cat", copy=True)
    np.testing.assert_array_equal(got, ref.nhood_count(g.indptr, g.indices, codes, 13).astype(np.float64))
    assert got.sum() == g.nnz
