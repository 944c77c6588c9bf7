"""The observed statistics of ligrec on a device-resident X (``sqb_ligrec_observed``, csrc/dense.cu), specified without a GPU:
the launch rule that picks the kernel's warps per block from the opt-in shared-memory limit, a data generator whose values
separate pandas' compensated group mean from plausible wrong kernels, and a check of the Kahan restatement against exact
rational arithmetic.  ``tests/test_gpu_ligrec_observed.py`` runs the kernel on this data at every side of the launch rule."""

from __future__ import annotations

import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest

from tests.device_attrs import H100_SMEM_OPTIN
from tests.test_ligrec_device_selection import kahan_group_mean

pytestmark = pytest.mark.filterwarnings("ignore:invalid value encountered:RuntimeWarning")  # inf - inf in the sums

STATIC_SMEM = 48 * 1024  # dynamic shared memory a launch gets without cudaFuncAttributeMaxDynamicSharedMemorySize
PER_CLUSTER_LANE = 2 * 8 + 4  # sum and compensation (double), positive count (int)
KINDS = ("cancel_bracket", "cancel_tile", "wide", "posinf", "neginf", "bothinf", "threshold")


def observed_warps(n_cls: int, optin: int) -> tuple[int, int, bool] | None:
    """``sqb_ligrec_observed``'s launch rule: ``per_warp = n_cls * 32 * (2 * sizeof(double) + sizeof(int))`` bytes of
    accumulators per warp, ``wpb = min(4, optin / per_warp)`` warps per block, ``smem = per_warp * wpb``, the opt-in attribute
    set when ``smem > 48 KB``.  Returns ``(wpb, smem, needs_attr)``, or ``None`` when one warp does not fit (the call is
    refused with SQB_ERR_UNSUPPORTED)."""
    per_warp = n_cls * 32 * PER_CLUSTER_LANE
    if per_warp > optin:
        return None
    wpb = min(4, optin // per_warp)
    smem = per_warp * wpb
    return wpb, smem, smem > STATIC_SMEM


def test_observed_warps_h100_boundaries():
    def rule(n):
        return observed_warps(n, H100_SMEM_OPTIN)

    assert rule(1) == (4, 4 * 640, False)
    assert rule(19) == (4, 48640, False) and rule(20) == (4, 51200, True)  # the opt-in attribute from 20 clusters up
    assert rule(90)[0] == 4 and rule(91)[0] == 3
    assert rule(121)[0] == 3 and rule(122)[0] == 2
    assert rule(181)[0] == 2 and rule(182)[0] == 1
    assert rule(363) == (1, 232320, True) and rule(364) is None
    # every warp count in between is a contiguous range of cluster counts
    wpbs = [rule(n)[0] for n in range(1, 364)]
    assert wpbs == sorted(wpbs, reverse=True) and set(wpbs) == {1, 2, 3, 4}


def observed_case(rng, n_cells: int, n_genes: int, n_cls: int, dtype=np.float64, threshold: float = 0.5):
    """Expression (``dtype``, NaN included) and cluster codes on which a wrong observed-statistics kernel shows.

    Extends the recipe of ``test_ligrec_device_selection._adversarial`` (wide dynamic range, zeros, NaN, ±inf, cancellation,
    a one-cell cluster) to any shape, and places the special values per cluster so that every cluster meets them.  Column
    kind ``KINDS[j % len(KINDS)]`` for gene ``j``:

    * ``cancel_bracket``: per cluster, in cell order, ``1e16, 1, ..., 1, -1e16`` -- a plain sum loses every 1;
    * ``cancel_tile``: per cluster, in cell order, ``1e16, 1, -1e16, 3, ...``;
    * ``wide``: ``N(0, 1) * 10^U{-8..7}`` with 30 % zeros, 5 % NaN (0 after ``fillna``), 3 % stored ``-0.0`` and 3 % positive
      subnormals (``v > 0`` counts them, ``v >= 0`` counts the zeros too); every other kind starts from it;
    * ``posinf`` / ``neginf``: +inf (-inf) as the first (second) cell of every third cluster;
    * ``bothinf``: +inf and -inf in clusters ``k % 3 == 0`` (NaN), +inf only in ``k % 3 == 1``, -inf only in ``k % 3 == 2``;
    * ``threshold``: exactly ``round(threshold * size)`` positive cells per cluster, so ``npos / size == threshold`` wherever
      ``threshold * size`` is an integer and ``>=`` and ``>`` disagree there.

    Every cluster is present; clusters ``n_cls // 2`` and ``n_cls - 1`` hold one cell."""
    tiny = np.finfo(dtype).smallest_subnormal
    x = rng.standard_normal((n_cells, n_genes)) * 10.0 ** rng.integers(-8, 8, (n_cells, n_genes))
    x[rng.random(x.shape) < 0.3] = 0.0
    x[rng.random(x.shape) < 0.05] = np.nan
    x[rng.random(x.shape) < 0.03] = -0.0
    sub = rng.random(x.shape) < 0.03
    x[sub] = tiny * rng.integers(1, 8, int(sub.sum()))
    single = {n_cls // 2, n_cls - 1} if n_cls >= 3 else set()
    multi = np.array([k for k in range(n_cls) if k not in single])
    codes = rng.choice(multi, n_cells)
    codes[rng.choice(n_cells, n_cls, replace=False)] = np.arange(n_cls)  # every cluster present, the singles once
    sizes = np.bincount(codes, minlength=n_cls)
    order = np.argsort(codes, kind="stable")
    rank = np.empty(n_cells, np.int64)
    rank[order] = np.arange(n_cells) - np.repeat(np.cumsum(sizes) - sizes, sizes)  # position of each cell in its cluster
    size = sizes[codes]
    kmod = codes % 3
    for j in range(n_genes):
        kind = KINDS[j % len(KINDS)]
        col = x[:, j]
        if kind == "cancel_bracket":
            col[:] = 1.0
            col[rank == 0] = 1e16
            col[(rank == size - 1) & (size >= 3)] = -1e16
        elif kind == "cancel_tile":
            col[:] = np.array([1e16, 1.0, -1e16, 3.0])[rank % 4]
        elif kind == "posinf":
            col[(rank == 0) & (kmod == 0) & (size >= 2)] = np.inf
        elif kind == "neginf":
            col[(rank == 1) & (kmod == 0)] = -np.inf
        elif kind == "bothinf":
            col[(rank == 0) & (kmod != 2) & (size >= 3)] = np.inf
            col[(rank == 1) & (kmod != 1)] = -np.inf
        elif kind == "threshold":
            npos = np.round(threshold * sizes)[codes]
            pos = np.where(rng.random(n_cells) < 0.3, tiny, rng.random(n_cells) + 0.5)
            non = rng.choice(np.array([0.0, -0.0, np.nan, -2.5]), n_cells)
            col[:] = np.where(rank < npos, pos, non)
    return x.astype(dtype), codes.astype(np.int32)


def pandas_group_mean(x0: np.ndarray, codes: np.ndarray, n_cls: int) -> np.ndarray:
    """What ``ligrec_analysis`` takes as the observed means: ``groupby('clusters', observed=True).mean()``."""
    df = pd.DataFrame(x0, columns=list(range(x0.shape[1])))
    df["clusters"] = pd.Categorical(codes, categories=list(range(n_cls)))
    return df.groupby("clusters", observed=True).mean().values


def group_sum(x0: np.ndarray, codes: np.ndarray, n_cls: int, *, compensated: bool, reset: bool = True) -> np.ndarray:
    """The group mean of a plain sequential sum (``compensated=False``) or of a Kahan sum with or without the NaN reset of its
    compensation: the wrong kernels the GPU tests must tell from pandas."""
    s = np.zeros((n_cls, x0.shape[1]))
    comp = np.zeros_like(s)
    with np.errstate(invalid="ignore"):
        for c in range(x0.shape[0]):
            k = codes[c]
            if not compensated:
                s[k] = s[k] + x0[c]
                continue
            y = x0[c] - comp[k]
            t = s[k] + y
            cp = (t - s[k]) - y
            comp[k] = np.where(np.isnan(cp), 0.0, cp) if reset else cp
            s[k] = t
    return s / np.bincount(codes, minlength=n_cls)[:, None].astype(np.float64)


def cluster_counts(b: np.ndarray, codes: np.ndarray, n_cls: int) -> np.ndarray:
    """True entries of the boolean ``b`` per (cluster, gene), exact: a float64 product of 0/1 matrices (counts far below
    2^53).  ``cluster_counts(x0 > 0, ...)`` is the positive count of the expression-fraction mask."""
    onehot = np.zeros((n_cls, b.shape[0]))
    onehot[codes, np.arange(b.shape[0])] = 1.0
    return (onehot @ b.astype(np.float64)).astype(np.int64)


def fill(x: np.ndarray) -> np.ndarray:
    """``fillna(0.0)`` in float64: what the gather writes with ``nan_zero``."""
    x0 = np.asarray(x, np.float64).copy()
    x0[np.isnan(x0)] = 0.0
    return x0


def kind_mask(n_genes: int, kind: str) -> np.ndarray:
    return np.array([KINDS[j % len(KINDS)] == kind for j in range(n_genes)])


@pytest.mark.parametrize("n_cls,n_cells,dtype", [(20, 3000, np.float64), (182, 3000, np.float64), (363, 3000, np.float64),
                                                 (91, 2730, np.float32)])
def test_data_discriminates(n_cls, n_cells, dtype):
    """The GPU tests compare the kernel with pandas; on this data a plain sum, a Kahan sum without the NaN reset and a
    ``v >= 0`` count all disagree with pandas, while the Kahan restatement agrees bit for bit."""
    x, codes = observed_case(np.random.default_rng(n_cls), n_cells, 31, n_cls, dtype)
    x0 = fill(x)
    expected = pandas_group_mean(x0, codes, n_cls)
    assert kahan_group_mean(x0, codes, n_cls).tobytes() == expected.tobytes()
    assert group_sum(x0, codes, n_cls, compensated=True).tobytes() == expected.tobytes()
    sizes = np.bincount(codes, minlength=n_cls)
    assert sizes.min() == 1 and (sizes == 1).sum() >= 2 and (sizes > 0).all()
    # a plain sequential sum differs from pandas on >= 20 % of all cells, and on the bracketed cancelling genes of every
    # cluster with at least four cells (with three, 1e16 + 1 - 1e16, Kahan loses the 1 as well)
    naive = group_sum(x0, codes, n_cls, compensated=False)
    differs = naive.view(np.uint64) != expected.view(np.uint64)
    assert differs.mean() >= 0.20, differs.mean()
    assert differs[sizes >= 4][:, kind_mask(31, "cancel_bracket")].all()
    # a more accurate sum differs too: on the tile genes (1e16, 1, -1e16, 3) Kahan loses the 1 when -1e16 + 1 rounds, so
    # pandas' mean is not the correctly rounded one (math.fsum) on >= 40 % of the clusters of four cells or more
    tile = np.flatnonzero(kind_mask(31, "cancel_tile"))
    exact = np.array([[math.fsum(x0[codes == k, j]) / sizes[k] for j in tile] for k in range(n_cls)])
    assert (exact != expected[:, tile])[sizes >= 4].mean() >= 0.4
    # Kahan without the NaN reset: NaN where pandas has +-inf
    no_reset = group_sum(x0, codes, n_cls, compensated=True, reset=False)
    lost = np.isinf(expected) & np.isnan(no_reset)
    assert lost.sum() >= n_cls // 3, lost.sum()
    assert np.isposinf(expected[lost]).any() and np.isneginf(expected[lost]).any()
    assert np.isnan(expected).any()  # +inf and -inf in one cluster
    # the positive count: subnormals count, -0.0 and zeros do not; the threshold genes sit exactly on the threshold
    assert (x0 > 0).sum() > 0 and ((x0 > 0) & (x0 < np.finfo(dtype).tiny)).any() and (np.signbit(x0) & (x0 == 0)).any()
    npos = cluster_counts(x0 > 0, codes, n_cls)
    assert (npos != cluster_counts(x0 >= 0, codes, n_cls)).mean() > 0.5  # v >= 0 counts the zeros
    frac = npos / sizes[:, None].astype(np.float64)
    on = (frac == 0.5)[:, kind_mask(31, "threshold")]
    assert on.sum() >= 3  # >= and > disagree here
    assert (frac >= 0.5).any() and (frac < 0.5).any()


def _exact_means(x0: np.ndarray, codes: np.ndarray, n_cls: int):
    """Exact rational sum, sum of absolute values and count per (cluster, gene) of the finite data."""
    n_genes = x0.shape[1]
    s = [[Fraction(0)] * n_genes for _ in range(n_cls)]
    a = [[Fraction(0)] * n_genes for _ in range(n_cls)]
    for c in range(x0.shape[0]):
        k = codes[c]
        for j in range(n_genes):
            v = Fraction(float(x0[c, j]))
            s[k][j] += v
            a[k][j] += abs(v)
    return s, a, np.bincount(codes, minlength=n_cls)


def _within_kahan_bound(got: float, exact_sum: Fraction, abs_sum: Fraction, n: int) -> bool:
    """``|got - S/n| <= (1 + eps) (2 eps + 2 n eps^2) sum|x| / n + eps |S/n| + 2^-1075``: the Kahan summation bound (Higham,
    Accuracy and Stability of Numerical Algorithms, 2nd ed., §4.3) carried through the rounded division, eps = 2^-53; the last
    term is the division's absolute error when the mean underflows (a subnormal sum over a count above 1).  Additions are
    exact in the subnormal range, so the sum needs no such term."""
    eps = Fraction(1, 2**53)
    mean = exact_sum / n
    bound = (1 + eps) * (2 * eps + 2 * n * eps * eps) * abs_sum / n + eps * abs(mean) + Fraction(1, 2**1075)
    return abs(Fraction(got) - mean) <= bound


@pytest.mark.parametrize("n_cls,n_cells", [(5, 400), (20, 600), (91, 700)])
def test_kahan_restatement_within_the_exact_bound(n_cls, n_cells):
    """An independent check of the restatement the GPU tests hold the kernel to: exact rational cluster sums, no shared
    arithmetic.  Every finite mean lies within the Kahan error bound of the exact mean; the plain sum breaks it on the
    bracketed cancelling genes.  Clusters with +-inf give what IEEE addition of those values gives: the infinity, or NaN."""
    x, codes = observed_case(np.random.default_rng(100 + n_cls), n_cells, 14, n_cls)
    x0 = fill(x)
    got = kahan_group_mean(x0, codes, n_cls)
    naive = group_sum(x0, codes, n_cls, compensated=False)
    fin = np.isfinite(x0)
    has_inf = cluster_counts(~fin, codes, n_cls) > 0  # clusters holding an infinity, per gene
    x_fin = np.where(fin, x0, 0.0)
    s, a, counts = _exact_means(x_fin, codes, n_cls)
    bracket = kind_mask(14, "cancel_bracket")
    broken = 0
    for k in range(n_cls):
        for j in range(14):
            if has_inf[k, j]:
                vals = x0[codes == k, j]
                pos, neg = np.isposinf(vals).any(), np.isneginf(vals).any()
                assert (np.isnan(got[k, j]) if pos and neg else got[k, j] == (np.inf if pos else -np.inf)), (k, j)
                continue
            assert _within_kahan_bound(got[k, j], s[k][j], a[k][j], counts[k]), (k, j, got[k, j], float(s[k][j] / counts[k]))
            if bracket[j] and counts[k] >= 8:
                assert not _within_kahan_bound(naive[k, j], s[k][j], a[k][j], counts[k]), (k, j)
                broken += 1
    assert broken >= n_cls // 2
