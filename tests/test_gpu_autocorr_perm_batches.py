"""GPU parity of Moran's I / Geary's C permutation scores across the batches of ``sqb_autocorr_run_perms``.

Permutations are staged in batches of at most 32; for sparse X one launch of ``ac_sparse_kernel<..., PERM=true>`` scores a
whole batch and writes permutation ``pb`` of the batch to ``out[pb * n_feat + g]``, the batch to ``out + p0 * n_feat``.  A
batch of 33 or 70 permutations therefore exercises every in-batch slot and the batch offsets.  Each row of
``score_perms`` must equal, bit for bit, the single-permutation score of the same permutation (the same fixed-order
reductions), and a sample of rows must match the oracle on ``W[idx, :]``."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from oracle import ref
from squidpy_b200._rng import spawn_generators
from squidpy_b200.gr import AutocorrPlan
from squidpy_b200.gr._ppatterns import _p_value_calc
from tools import synth

pytestmark = pytest.mark.gpu
TIGHT = dict(rtol=1e-10, atol=1e-13)
BATCH = 32  # permutations per device batch (autocorr.cu sqb_autocorr_run_perms)
ORACLE = {"moran": ref.morans_i, "geary": ref.gearys_c}


def batches(n_perms: int) -> list[int]:
    """``batch = n_perms < 32 ? n_perms : 32``; the last batch takes the rest."""
    b = min(n_perms, BATCH)
    return [min(b, n_perms - p0) for p0 in range(0, n_perms, b)]


def weight_format(w: sp.csr_matrix) -> str:
    """``sqb_autocorr_create``'s choice: rows of <= 7 entries sharing one float32 weight -> compact; other float32 rows of
    <= 8 / <= 16 entries -> 8 / 16 lanes per row; everything else (float64 weights, longer rows) -> CSR."""
    deg = np.diff(w.indptr).max()
    if w.data.dtype == np.float32 and deg <= 7:
        first = np.repeat(w.data[w.indptr[:-1]], np.diff(w.indptr))
        if (w.data.view(np.uint32) == first.view(np.uint32)).all():
            return "compact"
    if w.data.dtype == np.float32 and deg <= 8:
        return "lanes8"
    if w.data.dtype == np.float32 and deg <= 16:
        return "lanes16"
    return "csr"


def _weights(fmt: str, n_rows=50, n_cols=60) -> sp.csr_matrix:
    g = synth.hex_graph(n_rows, n_cols)
    if fmt == "compact":  # row-normalised lattice: <= 6 entries per row, all 1/deg
        from sklearn.preprocessing import normalize

        normalize(g, norm="l1", axis=1, copy=False)
        return g
    n = g.shape[0]
    rng = np.random.default_rng(1)
    deg = {"lanes8": 8, "lanes16": 13, "csr": 6}[fmt]
    cols = np.stack([rng.choice(n, deg, replace=False) for _ in range(n)])
    dt = np.float64 if fmt == "csr" else np.float32
    w = sp.csr_matrix((rng.random(n * deg).astype(dt), cols.ravel(), np.arange(0, n * deg + 1, deg)), shape=(n, n))
    w.sort_indices()
    return w


def _features(kind: str, n: int):
    if kind == "dense_f64":
        return np.random.default_rng(2).random((n, 40))
    x = sp.random(n, 40, density=0.15, format="csr", random_state=3, dtype=np.float64)
    x.data = np.round(x.data * 8) / 4 - 0.5  # negative values and explicit zeros among the stored entries
    return x.astype(np.float32) if kind == "sparse_f32" else x


def _xt(x):
    return x.T.tocsr() if sp.issparse(x) else np.ascontiguousarray(x.T)


@pytest.mark.parametrize("kind", ["sparse_f32", "sparse_f64", "dense_f64"])
@pytest.mark.parametrize("fmt", ["compact", "lanes8", "lanes16", "csr"])
@pytest.mark.parametrize("mode", ["moran", "geary"])
def test_score_perms_across_batches(mode, fmt, kind):
    w = _weights(fmt)
    assert weight_format(w) == fmt
    n = w.shape[0]
    x = _features(kind, n)
    plan = AutocorrPlan(w)
    plan.load(x, obs_major=True)
    rng = np.random.default_rng(70)
    idx = np.stack([rng.permutation(n) for _ in range(70)])
    single = np.stack([plan.score(mode, row_perm=idx[p]) for p in range(70)])
    assert np.isfinite(single).all()
    for P, split in ((32, [32]), (33, [32, 1]), (70, [32, 32, 6])):
        assert batches(P) == split
        got = plan.score_perms(mode, idx[:P])
        for p in range(P):
            np.testing.assert_array_equal(got[p], single[p], err_msg=f"P={P} row {p}")
    for p in (0, 15, 16, 31, 32, 69):  # both halves of a batch, the batch edges and the last row
        np.testing.assert_allclose(single[p], ORACLE[mode](w[idx[p], :], _xt(x)), **TIGHT)
    plan.close()


@pytest.mark.parametrize("mode", ["moran", "geary"])
def test_million_observations_global_bitmap_33_perms(mode):
    """1M observations: the bitmap of a feature no longer fits shared memory; 33 permutations take two batches."""
    from sklearn.preprocessing import normalize

    g = synth.hex_graph(1000, 1000)
    normalize(g, norm="l1", axis=1, copy=False)
    n = g.shape[0]
    x = sp.random(n, 6, density=0.05, format="csr", random_state=5, dtype=np.float32)
    plan = AutocorrPlan(g)
    plan.load(x, obs_major=True)
    rng = np.random.default_rng(33)
    idx = np.stack([rng.permutation(n) for _ in range(33)])
    got = plan.score_perms(mode, idx)
    for p in range(33):
        np.testing.assert_array_equal(got[p], plan.score(mode, row_perm=idx[p]), err_msg=f"row {p}")
    for p in (17, 32):
        np.testing.assert_allclose(got[p], ORACLE[mode](g[idx[p], :], x.T.tocsr()), **TIGHT)
    plan.close()


@pytest.mark.parametrize("mode", ["moran", "geary"])
def test_api_pval_sim_with_70_perms(mode):
    """``spatial_autocorr(n_perms=70)``: three device batches.  Its simulation p-values equal ``_p_value_calc`` applied to
    oracle scores of the same permutations (``spawn_generators(seed, 70)[p].permutation(n)``); this isolates the kernel
    from the p-value formula."""
    from sklearn.preprocessing import normalize

    g = synth.hex_graph(60, 67)
    n = g.shape[0]
    co = synth.hex_coords(60, 67)
    rng = np.random.default_rng(4)
    X = np.linspace(0.0, 0.1, 24) * np.sin(co[:, :1] / rng.uniform(200, 2000, 24)) + rng.normal(0, 1.0, (n, 24))  # weak signal
    ad = synth.make_adata(co, g, None, X=X)
    seed = 17
    df = sq.gr.spatial_autocorr(ad, mode=mode, n_perms=70, seed=seed, copy=True)
    w = g.copy()
    normalize(w, norm="l1", axis=1, copy=False)
    score = ORACLE[mode](w, X.T)
    gens = spawn_generators(seed, 70)
    sims = np.stack([ORACLE[mode](w[gens[p].permutation(n), :], X.T) for p in range(70)])
    params = {"mode": mode, "two_tailed": False, "expected": -1.0 / (n - 1) if mode == "moran" else 1.0}
    exp = _p_value_calc(score, sims, w, params)
    df = df.loc[list(ad.var_names)]
    np.testing.assert_allclose(df["I" if mode == "moran" else "C"].to_numpy(), score, **TIGHT)
    np.testing.assert_array_equal(df["pval_sim"].to_numpy(), exp["pval_sim"])
    assert len(np.unique(exp["pval_sim"])) > 3  # not all at one extreme
    np.testing.assert_allclose(df["var_sim"].to_numpy(), exp["var_sim"], rtol=1e-8)
