"""Moran's I / Geary's C on ill-conditioned and constant features, against the long-double definition.

The sparse per-feature kernel never visits the W rows of unstored observations: it recovers their share from the column
sums of W.  Those correction terms are not centred, and when every observation is stored they cancel down to rounding
noise times m^2 (m the feature's mean).  So the cases here are features whose mean is large next to their spread
(m/sigma up to 1e6), stored at every observation, at every observation but one, at about half and at one; on every
weight format of the sparse kernel, on the dense tiles, on row permutations, at 1M observations and from device memory.
Constant features (0.1, float32(0.1), 1/3, -7.3, 0) are the definition's 0/0 and must give NaN whether or not the
device's mean rounds back to the value.

Bounds: ``rtol = 1e-10`` where the field is autocorrelated (|I| >= 0.3, asserted through the reference) and
``|d| <= 1e-12 * autocorr_scale`` elsewhere (white noise, permuted W, sparse storage), where I is near 0 and a relative
bound means nothing; features stored at all observations but one keep the uncentred column-sum terms and are held to
``NEAR_FULL_KSCALE * scale + NEAR_FULL_ATOL``.  Every case first asserts which path it is on: stored count and weight
format."""

from __future__ import annotations

import functools

import numpy as np
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from oracle import ref
from squidpy_b200._rng import spawn_generators
from squidpy_b200.gr import AutocorrPlan
from squidpy_b200.gr._ppatterns import _p_value_calc
from tests import device_attrs
from tests import known_autocorr as ka
from tests.test_gpu_autocorr_perm_batches import weight_format
from tools import synth

pytestmark = pytest.mark.gpu
RTOL = 1e-10  # autocorrelated fields
KSCALE = 1e-12  # |d| <= KSCALE * autocorr_scale elsewhere
ROWS, COLS = 100, 200  # 20 000 spots
OFFSETS = {np.float64: (0.0, 1e2, 1e4, 1e6), np.float32: (0.0, 1e2, 1e4)}  # float32: quantum of 1e4 ~ 1e-3, far below sigma
STORAGE = ("full", "explicit_zeros", "all_but_one", "half", "single")
FORMATS = ("compact_rownorm", "compact_binary", "lanes8", "lanes16", "csr")
MODES = ("moran", "geary")


def _ring2(rows, cols):
    """Pairs two steps apart along a lattice row or column: with the 6 hex neighbours, up to 10 entries per row."""
    n = rows * cols
    r, c = np.divmod(np.arange(n), cols)
    src, dst = [], []
    for rr, cc in ((r, c - 2), (r, c + 2), (r - 2, c), (r + 2, c)):
        ok = (rr >= 0) & (rr < rows) & (cc >= 0) & (cc < cols)
        src.append(np.flatnonzero(ok))
        dst.append(rr[ok] * cols + cc[ok])
    return sp.csr_matrix((np.ones(sum(s.size for s in src), np.float32), (np.concatenate(src), np.concatenate(dst))), shape=(n, n))


@functools.lru_cache(maxsize=None)
def weights(fmt: str, rows: int = ROWS, cols: int = COLS) -> sp.csr_matrix:
    """Spatial weight matrices on the hex lattice (so that a smooth field is autocorrelated) in each format of
    ``ac_sparse_kernel``: compact 32-byte rows (FMT 3, row-normalised or binary), 8 lanes (FMT 0: <= 8 entries of random
    float32 weights), 16 lanes (FMT 1: <= 16) and CSR (FMT 2: float64 weights)."""
    from sklearn.preprocessing import normalize

    g = synth.hex_graph(rows, cols)
    if fmt == "compact_rownorm":
        normalize(g, norm="l1", axis=1, copy=False)
        return g
    if fmt == "compact_binary":
        return g
    if fmt == "lanes16":
        g = (g + _ring2(rows, cols)).tocsr()
    rng = np.random.default_rng(len(fmt))
    dt = np.float64 if fmt == "csr" else np.float32
    w = sp.csr_matrix((rng.uniform(0.5, 1.5, g.nnz).astype(dt), g.indices.astype(np.int32), g.indptr.astype(np.int32)), shape=g.shape)
    w.sort_indices()
    return w


EXPECTED_FORMAT = {"compact_rownorm": "compact", "compact_binary": "compact", "lanes8": "lanes8", "lanes16": "lanes16", "csr": "csr"}


def smooth_field(rows: int, cols: int, seed: int) -> np.ndarray:
    """Unit-variance field that varies over tens of lattice spacings, plus 30 % noise: |I| well above 0.3 on the lattice."""
    co = synth.hex_coords(rows, cols, scale=1.0)
    rng = np.random.default_rng(seed)
    f = np.sin(co[:, 0] / rng.uniform(8, 15) + rng.uniform(0, 6)) + np.cos(co[:, 1] / rng.uniform(8, 15) + rng.uniform(0, 6))
    f = f / f.std() + rng.normal(0.0, 0.3, f.size)
    return f / f.std()


@functools.lru_cache(maxsize=None)
def conditioning_matrix(dtype) -> tuple[sp.csr_matrix, tuple]:
    """Observations x features CSR: one feature per (offset, field, storage).  Returns the matrix and the case of every
    column (offset, field, storage, stored count)."""
    n = ROWS * COLS
    rng = np.random.default_rng(11)
    cols, cases = [], []
    for offset in OFFSETS[dtype]:
        for field in ("smooth", "white"):
            for storage in STORAGE:
                v = offset + (smooth_field(ROWS, COLS, len(cols)) if field == "smooth" else rng.normal(size=n))
                v = v.astype(dtype)
                assert (v != 0).all()
                if storage == "full":
                    idx = np.arange(n)
                elif storage == "explicit_zeros":
                    idx = np.arange(n)
                    v[rng.random(n) < 0.5] = 0.0
                elif storage == "all_but_one":
                    idx = np.delete(np.arange(n), rng.integers(n))
                elif storage == "half":
                    idx = np.flatnonzero(rng.random(n) < 0.5)
                else:
                    idx = rng.integers(n, size=1)
                cols.append(sp.csc_matrix((v[idx], idx, [0, idx.size]), shape=(n, 1)))
                cases.append((offset, field, storage, idx.size))
    x = sp.hstack(cols, format="csr")
    assert x.dtype == dtype
    return x, tuple(cases)


def _ref(w, x) -> tuple[np.ndarray, np.ndarray]:
    """(I, C) and their error scales for every column of x (observations x features)."""
    xd = x.toarray() if sp.issparse(x) else np.asarray(x)
    vals = np.array([ka.sparse_longdouble(w, xd[:, k]) for k in range(xd.shape[1])])
    scales = np.array([ka.autocorr_scale(w, xd[:, k]) for k in range(xd.shape[1])])
    return vals, scales


@functools.lru_cache(maxsize=None)
def reference(fmt: str, dtype) -> tuple[np.ndarray, np.ndarray]:
    return _ref(weights(fmt), conditioning_matrix(dtype)[0])


def assert_case(got, exp, scale, autocorrelated, what, k=KSCALE, atol=0.0):
    d = np.abs(got - exp)
    if autocorrelated:
        assert d <= RTOL * abs(exp), f"{what}: got {got!r}, ref {exp!r}, rel {d / abs(exp):.3g}"
    else:
        assert d <= k * scale + atol, f"{what}: got {got!r}, ref {exp!r}, |d| {d:.3g} > {k:g} * scale {scale:.3g} + {atol:.3g}"


# A feature stored at all observations but one still takes the column-sum formulation (see autocorr.cu): its correction
# terms are not centred.  Moran's m^2 * (S0 - E) carries the rounding of S0 and E (about N * eps * S0 for float64 weights)
# over sum z^2 >= m^2, an absolute error of order N * eps in I whatever m is; the other terms cancel to at most
# 1.6e-11 * scale on this suite.  Measured on an H100 at N = 20 000: 1.95e-11 (Moran, float64 weights, m/sigma = 1e4).
# These bounds pin that accuracy; features stored everywhere or at half the observations meet KSCALE * scale.
NEAR_FULL_KSCALE = 5e-11
NEAR_FULL_ATOL = 8 * ROWS * COLS * np.finfo(np.float64).eps  # 3.6e-11


def check_scores(got, exp, scale, cases, mode, what, autocorrelated_ok=True):
    k = MODES.index(mode)
    n = ROWS * COLS
    for f, (offset, field, storage, stored) in enumerate(cases):
        assert stored == {"full": n, "explicit_zeros": n, "all_but_one": n - 1}.get(storage, stored) and (storage != "half" or stored < n)
        auto = autocorrelated_ok and field == "smooth" and storage == "full"  # a zero among values near m dominates sum z^2
        if auto:
            assert abs(exp[f, 0]) >= 0.3  # the case is the one it claims to be
        assert_case(got[f], exp[f, k], scale[f, k], auto, f"{what} {mode} feature {f} (m={offset:g}, {field}, {storage}, {stored} stored)",
                    **(dict(k=NEAR_FULL_KSCALE, atol=NEAR_FULL_ATOL) if storage == "all_but_one" else {}))


# ---------------------------------------------------------------------------------------------------------------------
# sparse per-feature kernel: every weight format, float32 / float64 X, unpermuted and a batch of 33 permutations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
def test_sparse_offsets_and_storage(mode, fmt, dtype):
    w = weights(fmt)
    assert weight_format(w) == EXPECTED_FORMAT[fmt]
    x, cases = conditioning_matrix(dtype)
    exp, scale = reference(fmt, dtype)
    plan = AutocorrPlan(w)
    plan.load(x, obs_major=True)
    check_scores(plan.score(mode), exp, scale, cases, mode, f"{fmt}/{np.dtype(dtype).name}")
    plan.close()


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("mode", MODES)
def test_sparse_permutations(mode, fmt):
    """``score_perms`` on 33 row permutations (two batches) against the definition on ``W[idx, :]``."""
    w = weights(fmt)
    assert weight_format(w) == EXPECTED_FORMAT[fmt]
    x, cases = conditioning_matrix(np.float64)
    n = w.shape[0]
    rng = np.random.default_rng(33)
    idx = np.stack([rng.permutation(n) for _ in range(33)])
    plan = AutocorrPlan(w)
    plan.load(x, obs_major=True)
    got = plan.score_perms(mode, idx)
    plan.close()
    for p in (0, 31, 32):
        exp, scale = _ref(w[idx[p], :], x)
        check_scores(got[p], exp, scale, cases, mode, f"{fmt} perm {p}", autocorrelated_ok=False)


@functools.lru_cache(maxsize=None)
def _switch_perms() -> np.ndarray:
    rng = np.random.default_rng(5)
    return np.stack([rng.permutation(ROWS * COLS) for _ in range(2)])


@functools.lru_cache(maxsize=None)
def _perm_reference(fmt: str, p: int):
    return _ref(weights(fmt)[_switch_perms()[p], :], conditioning_matrix(np.float64)[0])


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("first,then", [("moran", "geary"), ("geary", "moran")])
def test_permutations_after_the_other_mode(first, then, fmt):
    """The per-feature terms a permuted pass reuses (mean, sum z^2, the column-sum terms) are written by the last unpermuted
    pass, whichever its mode: after ``score(first)`` a plan must score ``then`` on permutations, through ``score_perms`` and
    ``score(row_perm=...)``, as the definition on ``W[idx, :]`` says."""
    w = weights(fmt)
    assert weight_format(w) == EXPECTED_FORMAT[fmt]
    x, cases = conditioning_matrix(np.float64)
    idx = _switch_perms()
    plan = AutocorrPlan(w)
    plan.load(x, obs_major=True)
    plan.score(first)
    batch = plan.score_perms(then, idx)
    plan.score(first)
    single = plan.score(then, row_perm=idx[0])
    plan.close()
    for p, got in ((0, batch[0]), (1, batch[1]), (0, single)):
        exp, scale = _perm_reference(fmt, p)
        check_scores(got, exp, scale, cases, then, f"{fmt} {first} then {then} perm {p}", autocorrelated_ok=False)


# ---------------------------------------------------------------------------------------------------------------------
# dense tiles, device input, 1M observations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("fmt", ["compact_rownorm", "csr"])
@pytest.mark.parametrize("mode", MODES)
def test_dense_tiles_offsets(mode, fmt, dtype):
    w = weights(fmt)
    x, cases = conditioning_matrix(dtype)
    exp, scale = reference(fmt, dtype)
    xd = x.toarray()
    plan = AutocorrPlan(w)
    plan.load(xd, obs_major=True)
    got = plan.score(mode)
    check_scores(got, exp, scale, cases, mode, f"dense obs-major {fmt}/{np.dtype(dtype).name}")
    plan.load(np.ascontiguousarray(xd.T), obs_major=False)
    np.testing.assert_array_equal(plan.score(mode), got)  # feature-major tiles: the same fixed-order sums
    plan.close()


def test_device_sparse_csr_int32():
    """A torch ``sparse_csr`` tensor with int32 indices reaches the same kernel: scores equal the host load bit for bit."""
    import torch

    w = weights("compact_rownorm")
    x, cases = conditioning_matrix(np.float64)
    exp, scale = reference("compact_rownorm", np.float64)
    dev = torch.sparse_csr_tensor(torch.from_numpy(x.indptr.astype(np.int32)), torch.from_numpy(x.indices.astype(np.int32)),
                                  torch.from_numpy(x.data), size=x.shape).cuda()
    assert dev.crow_indices().dtype == torch.int32 and dev.col_indices().dtype == torch.int32
    plan = AutocorrPlan(w)
    for mode in MODES:
        plan.load(x, obs_major=True)
        host = plan.score(mode)
        plan.load(dev, obs_major=True)
        got = plan.score(mode)
        np.testing.assert_array_equal(got, host)
        check_scores(got, exp, scale, cases, mode, "device csr")
    plan.close()


def test_million_observations_fully_stored_offset():
    """1M observations (the bitmap lives in global scratch): a fully stored feature at m/sigma = 1e6 next to a sparse one."""
    g = weights("compact_rownorm", 1000, 1000)
    n = g.shape[0]
    rng = np.random.default_rng(6)
    full = 1e6 + smooth_field(1000, 1000, 3)
    sparse_col = np.where(rng.random(n) < 0.05, rng.normal(size=n), 0.0)
    x = sp.csr_matrix(np.stack([full, sparse_col], axis=1))
    assert np.diff(x.tocsc().indptr)[0] == n
    # the feature's bitmap (8 bytes per 32 observations) exceeds the shared memory a CTA may opt into, less the 4 KB the
    # kernels keep for static shared memory (ac_geometry): the global-scratch branch
    assert (n + 31) // 32 * 8 > device_attrs.smem_optin() - 4096
    exp = np.array([ka.sparse_longdouble(g, full), ka.sparse_longdouble(g, sparse_col)])
    scale = np.array([ka.autocorr_scale(g, full), ka.autocorr_scale(g, sparse_col)])
    assert abs(exp[0, 0]) >= 0.3
    plan = AutocorrPlan(g)
    plan.load(x, obs_major=True)
    for k, mode in enumerate(MODES):
        got = plan.score(mode)
        assert_case(got[0], exp[0, k], scale[0, k], True, f"1M full {mode}")
        assert_case(got[1], exp[1, k], scale[1, k], False, f"1M sparse {mode}")
    plan.close()


# ---------------------------------------------------------------------------------------------------------------------
# constant features: NaN on every path
# ---------------------------------------------------------------------------------------------------------------------
CONSTANTS = (0.1, float(np.float32(0.1)), 1.0 / 3.0, -7.3, 0.0)


@pytest.mark.parametrize("rows,cols", [(40, 50), (100, 200)], ids=["n2000", "n20000"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_constant_features_are_nan(rows, cols, dtype):
    """Every value equal is 0/0 in the definition.  Each constant is stored at every observation (the value 0 as explicit
    zeros); a last column, one ulp off a constant, must stay finite."""
    w = weights("compact_rownorm", rows, cols)
    n = w.shape[0]
    vals = [np.full(n, v, dtype=dtype) for v in CONSTANTS]
    near = np.full(n, dtype(0.1))
    near[n // 2] = np.nextafter(dtype(0.1), dtype(1))
    xd = np.stack(vals + [near], axis=1)
    idx = np.arange(n)
    x = sp.csr_matrix((xd.ravel(), np.tile(np.arange(xd.shape[1]), n), np.arange(0, xd.size + 1, xd.shape[1])), shape=xd.shape)
    assert x.nnz == xd.size and (x.getnnz(axis=0) == n).all()  # stored everywhere, the zeros too
    assert np.isfinite(ka.sparse_longdouble(w, near)).all() and all(np.isnan(ka.sparse_longdouble(w, v)).all() for v in vals)
    rng = np.random.default_rng(1)
    perms = np.stack([rng.permutation(n) for _ in range(3)])
    plan = AutocorrPlan(w)
    for m, what in ((x, "sparse"), (xd, "dense")):
        plan.load(m, obs_major=True)
        for mode in MODES:
            for got in (plan.score(mode), plan.score(mode, row_perm=idx[::-1]), *plan.score_perms(mode, perms)):
                assert np.isnan(got[:-1]).all(), f"{what} {mode}: {got[:-1]}"
                assert np.isfinite(got[-1]), f"{what} {mode}: near-constant feature gave {got[-1]}"
    plan.close()


# ---------------------------------------------------------------------------------------------------------------------
# the public API with permutations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_api_offset_feature_scores_and_pval_sim(mode):
    """``spatial_autocorr(n_perms=20)`` on a CSR X whose first feature is stored everywhere at m/sigma = 1e6: the scores
    match the definition and the simulation p-values equal those of the oracle's permuted scores (same seed)."""
    from sklearn.preprocessing import normalize

    rows, cols = 60, 67
    g = synth.hex_graph(rows, cols)
    n = g.shape[0]
    rng = np.random.default_rng(8)
    X = np.where(rng.random((n, 8)) < 0.2, rng.normal(size=(n, 8)) + 2.0, 0.0)
    X[:, 0] = 1e6 + smooth_field(rows, cols, 0)
    X[:, 1] = 1e4 + rng.normal(size=n)
    ad = synth.make_adata(synth.hex_coords(rows, cols), g, None, X=sp.csr_matrix(X))
    assert ad.X.getnnz(axis=0)[0] == n and ad.X.getnnz(axis=0)[1] == n
    seed, n_perms = 23, 20
    df = sq.gr.spatial_autocorr(ad, mode=mode, n_perms=n_perms, seed=seed, copy=True)
    w = g.copy()
    normalize(w, norm="l1", axis=1, copy=False)
    k = MODES.index(mode)
    score = np.array([ka.sparse_longdouble(w, X[:, f])[k] for f in range(X.shape[1])])
    scale = np.array([ka.autocorr_scale(w, X[:, f])[k] for f in range(X.shape[1])])
    assert abs(ka.sparse_longdouble(w, X[:, 0])[0]) >= 0.3
    gens = spawn_generators(seed, n_perms)
    oracle = ref.morans_i if mode == "moran" else ref.gearys_c
    sims = np.stack([oracle(w[gens[p].permutation(n), :], X.T) for p in range(n_perms)])
    assert (np.abs(sims - score) > 1e-9 * np.abs(score)).all()  # no comparison sits within rounding of the observed score
    params = {"mode": mode, "two_tailed": False, "expected": -1.0 / (n - 1) if mode == "moran" else 1.0}
    exp = _p_value_calc(score, sims, w, params)
    df = df.loc[list(ad.var_names)]
    got = df["I" if mode == "moran" else "C"].to_numpy()
    for f in range(X.shape[1]):
        assert_case(got[f], score[f], scale[f], f == 0, f"api {mode} feature {f}")
    np.testing.assert_array_equal(df["pval_sim"].to_numpy(), exp["pval_sim"])
