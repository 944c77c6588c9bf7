"""GPU parity of the pair histograms (co_occurrence float32, Ripley pair counts float64) beyond the lane-private limit.

``pairs_kernel`` keeps either one histogram column per lane (``LANEPRIV``: plain read-modify-write) or, when that does not
fit the block's opt-in shared memory, one histogram per warp updated with shared-memory atomics.  The second variant is
reached by ordinary arguments (``co_occurrence`` with >= 215 interval edges, ``ripley(n_steps >= 205)``), so both are
compared here with the brute-force oracle at the sizes where the branch changes, at the tile edges and at threshold shapes
that stress the first-bin lookup table.  Counts are integers: every comparison is exact."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest

import squidpy_b200 as sq
from oracle import ref
from squidpy_b200.gr import cooc_counts, pair_counts
from tests.device_attrs import H100_SMEM_OPTIN, smem_optin
from tools import synth

pytestmark = pytest.mark.gpu

PAIRS_THREADS, PAIRS_JCHUNK, PAIRS_NC = 256, 1024, 1024


def lane_private(L: int, itemsize: int, optin: int) -> bool:
    """The dispatch rule of ``pairs_run`` (pairs.cu), for float (itemsize 4) or double (8) coordinates:

        base_smem = PAIRS_JCHUNK * sizeof(V2) + (size_t)((L + 2) / 2 * 2) * sizeof(FT) + PAIRS_NC * sizeof(int);
        priv_smem = base_smem + (size_t)(PAIRS_THREADS / 32) * L * 32 * 4;
        lanepriv = priv_smem + 1024 <= c->smem_optin;
    """
    base = PAIRS_JCHUNK * 2 * itemsize + (L + 2) // 2 * 2 * itemsize + PAIRS_NC * 4
    return base + (PAIRS_THREADS // 32) * L * 32 * 4 + 1024 <= optin


@pytest.fixture(scope="module")
def optin():
    return smem_optin()


def _variant(L, itemsize, optin, expect_lanepriv, near_boundary):
    """Skip a case that straddles the boundary on a device with another opt-in limit; otherwise assert the branch it takes."""
    if near_boundary and optin != H100_SMEM_OPTIN:
        pytest.skip(f"boundary case written for {H100_SMEM_OPTIN} B of opt-in shared memory per block, this device has {optin} B")
    assert lane_private(L, itemsize, optin) == expect_lanepriv, (L, itemsize, optin)


def test_dispatch_rule_boundaries_on_h100():
    """On an H100 (232 448 B per block) float L <= 213 and double S <= 204 are lane-private."""
    assert lane_private(213, 4, H100_SMEM_OPTIN) and not lane_private(214, 4, H100_SMEM_OPTIN)
    assert lane_private(204, 8, H100_SMEM_OPTIN) and not lane_private(205, 8, H100_SMEM_OPTIN)


def _cooc_case(n, k, L, seed):
    rng = np.random.default_rng(seed)
    pts = (rng.random((n, 2)) * 500).astype(np.float32)
    labs = rng.integers(0, k, n).astype(np.int32)
    labs[labs == 1] = 0  # an empty label
    thr = np.sort(rng.random(L).astype(np.float32) * 400.0) ** 2
    thr[3] = thr[2]  # a repeated radius
    return pts, labs, thr


def _check_cooc(got, exp):
    np.testing.assert_array_equal(got, exp)
    np.testing.assert_array_equal(got, got.transpose(1, 0, 2))
    assert (np.diff(got, axis=2) >= 0).all()


@pytest.mark.parametrize("use_fma", [True, False])
@pytest.mark.parametrize("L,lanepriv,near", [(213, True, True), (214, False, True), (300, False, False), (4096, False, False)])
def test_cooc_vs_oracle_across_histogram_variants(optin, L, lanepriv, near, use_fma):
    _variant(L, 4, optin, lanepriv, near)
    k = 5
    pts, labs, thr = _cooc_case(3000, k, L, seed=L)
    exp = ref.occur_count(pts[:, 0], pts[:, 1], thr, labs, k, use_fma=use_fma)
    assert (exp[..., -1] > exp[..., -2]).any()  # the last radius adds pairs: a dropped last bin would show
    assert (exp[1] == 0).all() and (exp[:, 1] == 0).all()
    _check_cooc(cooc_counts(pts[:, 0], pts[:, 1], thr, labs, k, use_fma=use_fma), exp)


def _lattice_pair_counts(side, S):
    """Ordered pairs (self pairs included) of the side x side integer lattice within radius sqrt(m), m = 0 .. S-1.  Offsets
    (dx, dy) occur (side - |dx|) (side - |dy|) times and d2 = dx^2 + dy^2 is an integer, so sqrt(d2) <= sqrt(m) iff
    d2 <= m (sqrt is correctly rounded and strictly increasing on integers): every radius has pairs exactly on it."""
    d = np.arange(-(side - 1), side)
    d2 = (d[:, None] ** 2 + d[None, :] ** 2).ravel()
    w = ((side - np.abs(d))[:, None] * (side - np.abs(d))[None, :]).ravel()
    return np.cumsum(np.bincount(d2, weights=w, minlength=S))[:S].astype(np.int64)


@pytest.mark.parametrize("S,lanepriv,near", [(204, True, True), (205, False, True), (400, False, False), (4096, False, False)])
def test_pair_counts_vs_oracle_across_histogram_variants(optin, S, lanepriv, near):
    _variant(S, 8, optin, lanepriv, near)
    rng = np.random.default_rng(S)
    groups = [rng.random((m, 2)) * 1000 for m in (1500, 0, 1, 2200)]
    sup = np.sort(rng.random(S) * 900)
    sup[5] = sup[4]
    exp = np.stack([ref.pair_counts(g, sup) if len(g) else np.zeros(S, np.int64) for g in groups])
    assert (exp[:, -1] > exp[:, -2]).any()
    got = pair_counts(groups, sup)
    np.testing.assert_array_equal(got, exp)
    parts = [pair_counts(groups, sup, shard=(r, 3)) for r in range(3)]
    np.testing.assert_array_equal(sum(parts), exp)  # tile shards add up (multi-GPU path)
    gx, gy = np.meshgrid(np.arange(60), np.arange(60))
    lattice = np.stack([gx.ravel(), gy.ravel()], 1).astype(np.float64)
    lsup = np.sqrt(np.arange(S, dtype=np.float64))
    lexp = _lattice_pair_counts(60, S)
    if S < 300:
        np.testing.assert_array_equal(lexp, ref.pair_counts(lattice, lsup))  # the closed form agrees with brute force
    assert (np.diff(lexp) > 0).sum() > S // 10  # many radii are lattice distances: pairs exactly on the radius
    np.testing.assert_array_equal(pair_counts([lattice], lsup)[0], lexp)
    np.testing.assert_array_equal(sum(pair_counts([lattice], lsup, shard=(r, 3))[0] for r in range(3)), lexp)


# group sizes around the 1024-point tile (same-group 1024 x 1024 upper-triangle tiles, weight 2 off the diagonal) and the
# 4096-point column tile of cross-group tiles, with empty groups between them
TILE_SIZES = (1023, 0, 1024, 1025, 0, 4095, 4096, 4097)


@pytest.mark.parametrize("L,lanepriv", [(213, True), (214, False)])
def test_cooc_tile_edges(optin, L, lanepriv):
    _variant(L, 4, optin, lanepriv, True)
    rng = np.random.default_rng(11)
    labs = np.repeat(np.arange(len(TILE_SIZES), dtype=np.int32), TILE_SIZES)
    labs = labs[rng.permutation(labs.size)]
    n = labs.size
    pts = (rng.random((n, 2)) * 300).astype(np.float32)
    thr = np.sort(rng.random(L).astype(np.float32) * 250.0) ** 2
    thr[-1] = 2 * 300.0**2 + 1.0  # the largest radius holds every pair
    got = cooc_counts(pts[:, 0], pts[:, 1], thr, labs, len(TILE_SIZES))
    _check_cooc(got, ref.occur_count(pts[:, 0], pts[:, 1], thr, labs, len(TILE_SIZES)))
    sizes = np.array(TILE_SIZES)
    np.testing.assert_array_equal(got[..., -1], sizes[:, None] * sizes[None, :] - np.diag(sizes))  # ordered pairs i != j


@pytest.mark.parametrize("S,lanepriv", [(204, True), (205, False)])
def test_pair_counts_tile_edges(optin, S, lanepriv):
    _variant(S, 8, optin, lanepriv, True)
    rng = np.random.default_rng(12)
    groups = [rng.random((m, 2)) * 400 for m in TILE_SIZES]
    sup = np.concatenate([np.sort(rng.random(S - 1) * 300), [600.0]])
    exp = np.stack([ref.pair_counts(g, sup) if len(g) else np.zeros(S, np.int64) for g in groups])
    np.testing.assert_array_equal(exp[:, -1], np.array(TILE_SIZES) ** 2)  # every ordered pair, self pairs included
    np.testing.assert_array_equal(pair_counts(groups, sup), exp)


def _thresholds(shape, L):
    if shape == "geometric":  # 12 decades: most thresholds fall into the first lookup cell
        return (np.logspace(-12, 0, L) * 300.0**2).astype(np.float32)
    if shape == "equal":
        return np.full(L, 50.0**2, np.float32)
    if shape == "zero_first":
        t = np.sort(np.random.default_rng(L).random(L).astype(np.float32) * 200.0) ** 2
        t[:3] = 0.0
        return t
    if shape == "all_zero":
        return np.zeros(L, np.float32)
    raise AssertionError(shape)


@pytest.mark.parametrize("shape", ["geometric", "equal", "zero_first", "all_zero"])
@pytest.mark.parametrize("L,lanepriv,near", [(213, True, True), (300, False, False)])
def test_cooc_threshold_shapes(optin, shape, L, lanepriv, near):
    _variant(L, 4, optin, lanepriv, near)
    rng = np.random.default_rng(21)
    base = (rng.random((1200, 2)) * 400).astype(np.float32)
    pts = np.concatenate([base, base[:300], base[:100]])  # coincident points: distance exactly 0
    labs = rng.integers(0, 4, pts.shape[0]).astype(np.int32)
    thr = _thresholds(shape, L)
    exp = ref.occur_count(pts[:, 0], pts[:, 1], thr, labs, 4)
    assert exp[..., 0].sum() > 0  # the smallest radius (0 in three of the shapes) catches the coincident pairs
    _check_cooc(cooc_counts(pts[:, 0], pts[:, 1], thr, labs, 4), exp)
    _check_cooc(cooc_counts(pts[:, 0], pts[:, 1], thr, labs, 4, use_fma=False), ref.occur_count(pts[:, 0], pts[:, 1], thr, labs, 4, use_fma=False))


@pytest.mark.parametrize("shape", ["geometric", "equal", "zero_first", "negative_and_inf"])
@pytest.mark.parametrize("S,lanepriv,near", [(204, True, True), (400, False, False)])
def test_pair_counts_support_shapes(optin, shape, S, lanepriv, near):
    _variant(S, 8, optin, lanepriv, near)
    rng = np.random.default_rng(22)
    base = rng.random((1500, 2)) * 400
    pts = np.concatenate([base, base[:200]])
    if shape == "geometric":
        sup = np.logspace(-6, 0, S) * 300.0  # 12 decades in d2
    elif shape == "equal":
        sup = np.full(S, 50.0)
    elif shape == "zero_first":
        sup = np.sort(rng.random(S) * 200.0)
        sup[:3] = 0.0
    else:  # negative radii (internal threshold -1: nothing) and +inf (internal threshold DBL_MAX: everything)
        sup = np.sort(rng.random(S) * 200.0)
        sup[:4] = [-5.0, -1.0, -1.0, 0.0]
        sup[-2:] = np.inf
    exp = ref.pair_counts(pts, sup)
    if shape == "negative_and_inf":
        assert (exp[:3] == 0).all() and exp[3] == pts.shape[0] + 2 * 200 and (exp[-2:] == pts.shape[0] ** 2).all()
    np.testing.assert_array_equal(pair_counts([pts], sup)[0], exp)


def test_largest_histogram_is_accepted_and_one_more_is_refused():
    rng = np.random.default_rng(3)
    pts = (rng.random((500, 2)) * 100).astype(np.float32)
    labs = rng.integers(0, 3, 500).astype(np.int32)
    thr = np.sort(rng.random(4096).astype(np.float32) * 120.0) ** 2
    np.testing.assert_array_equal(cooc_counts(pts[:, 0], pts[:, 1], thr, labs, 3), ref.occur_count(pts[:, 0], pts[:, 1], thr, labs, 3))
    with pytest.raises(ValueError, match=r"L=4097 out of range \[1,4096\]"):
        cooc_counts(pts[:, 0], pts[:, 1], np.sort(rng.random(4097).astype(np.float32)), labs, 3)
    p64 = pts.astype(np.float64)
    sup = np.sort(rng.random(4096) * 120.0)
    np.testing.assert_array_equal(pair_counts([p64], sup)[0], ref.pair_counts(p64, sup))
    with pytest.raises(ValueError, match=r"S=4097 out of range \[1,4096\]"):
        pair_counts([p64], np.sort(rng.random(4097)))


def test_api_co_occurrence_301_edges(optin):
    """``co_occurrence`` with 301 interval edges (300 radii: the shared-atomics histogram) against the oracle's
    ``_co_occurrence_helper``."""
    assert not lane_private(300, 4, optin)
    rng = np.random.default_rng(8)
    n = 4000
    co = (rng.random((n, 2)) * 2000.0).astype(np.float32)
    codes = rng.integers(0, 6, n)
    lab = pd.Series(pd.Categorical.from_codes(codes, categories=[f"c{i}" for i in range(6)]))
    ad = synth.make_adata(co.astype(np.float64), None, lab)
    interval = np.linspace(5.0, 1200.0, 301)
    occ, iv = sq.gr.co_occurrence(ad, "cluster", interval=interval, copy=True)
    assert occ.shape == (6, 6, 300) and iv.dtype == np.float32
    exp_occ, _ = ref.co_occurrence_helper(co[:, 0], co[:, 1], iv, codes.astype(np.int32))
    np.testing.assert_allclose(occ, exp_occ, rtol=1e-12)
