"""CPU specification of the post-processors' device arithmetic (csrc/graph_device.cu) on a caller's graph:

* ``percentile_step``: the threshold from the device's radix-sorted distances, restated here from ``percentile_linear`` /
  ``percentile_linear_f32`` (two order statistics, numpy's ``linear`` method, float32 arithmetic for float32 distances as
  NEP 50 casts the Python percentile) plus the NaN rule, equals ``np.percentile`` of the same values for every size from 1 to
  4 096, sizes around 2^24 (where the float32 virtual index rounds), a fine grid of percentiles and data with NaN (either
  sign), +-inf and signed zeros;
* ``spectral``: the host's ``a.sum(axis=0)`` of a float32 CSR is a float32 sum of every column from 0 in row order, the
  order the device's column sums follow.
"""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

F32, F64 = np.float32, np.float64


def radix_order(v: np.ndarray) -> np.ndarray:
    """The values as float64 in cub's ascending radix order: by bit pattern with the sign flipped, so a NaN with its sign bit set
    comes first, -0.0 before +0.0, and any other NaN last."""
    d = np.asarray(v, dtype=F64)
    bits = d.view(np.uint64)
    key = np.where(bits >> np.uint64(63), ~bits, bits | np.uint64(1 << 63))
    return d[np.argsort(key, kind="stable")]


def percentile_linear(q: float, s: np.ndarray) -> float:
    """``percentile_linear``: float64 arithmetic on the two order statistics around (m - 1) q / 100."""
    m = s.size
    vi = (m - 1) * (q / 100.0)
    prev = np.floor(vi)
    ip = int(prev)
    nx = ip + 1
    if vi >= m - 1:  # numpy's index -1; gamma is computed from it
        ip = nx = m - 1
        prev = -1.0
    gamma = vi - prev
    a, b = F64(s[ip]), F64(s[nx])
    with np.errstate(invalid="ignore", over="ignore"):
        diff = b - a
        r = a + diff * F64(gamma)
        if gamma >= 0.5:
            r = b - diff * (F64(1.0) - F64(gamma))
    return float(r)


def percentile_linear_f32(q: float, s: np.ndarray) -> float:
    """``percentile_linear_f32``: q, the virtual index, its fraction and the interpolation in float32."""
    m = s.size
    qf = F32(q) / F32(100.0)
    vi = F32(m - 1) * qf
    ip = int(np.floor(vi))
    nx = ip + 1
    gamma = F32(vi - F32(ip))
    if vi >= F32(m - 1):
        ip = nx = m - 1
        gamma = F32(F64(vi) + 1.0)
    a, b = F32(s[ip]), F32(s[nx])
    with np.errstate(invalid="ignore", over="ignore"):
        diff = F32(b - a)
        r = F32(a + diff * gamma)
        if gamma >= F32(0.5):
            r = F32(b - diff * (F32(1.0) - gamma))
    return float(r)


def device_threshold(values: np.ndarray, q: float, sorted_=None) -> float:
    """``percentile_step``'s threshold: NaN when the first or the last radix-sorted value is NaN, else the two-statistic
    formula of the distances' dtype."""
    s = radix_order(values) if sorted_ is None else sorted_
    if np.isnan(s[0]) or np.isnan(s[-1]):
        return float("nan")
    return (percentile_linear_f32 if values.dtype == F32 else percentile_linear)(q, s)


def numpy_threshold(values: np.ndarray, q: float) -> float:
    with np.errstate(invalid="ignore", over="ignore"):
        return float(np.percentile(values, q))


def same(got: float, want: float) -> bool:
    """Equal, or both NaN.  The sign of a zero threshold is not compared: numpy's partition orders -0.0 and +0.0 as equal, and
    `dst > -0.0` marks what `dst > 0.0` marks."""
    return got == want or (np.isnan(got) and np.isnan(want))


Q_FINE = sorted({0.0, 37.5, 50.0, 90.0, 100.0, *np.round(np.linspace(0.0, 100.0, 81), 4).tolist(), 1e-7, 33.333333, 66.67, 99.9, 99.99999})
Q_COARSE = [0.0, 33.333333, 37.5, 50.0, 90.0, 99.99999, 100.0]


KINDS = ["finite", "signed_zeros", "inf", "inf_max", "nan", "neg_nan", "neg_inf"]


def _values(rng, m: int, dtype, kind: str) -> np.ndarray:
    v = rng.uniform(0.0, 10.0, m).astype(dtype)
    v[rng.random(m) < 0.2] = v[0]  # ties
    v[rng.random(m) < 0.1] = 0.0
    if kind == "signed_zeros":
        v[rng.random(m) < 0.3] = -0.0
    elif kind == "inf":
        v[rng.random(m) < 0.25] = np.inf
    elif kind == "inf_max":
        v[rng.integers(m)] = np.inf
    elif kind == "nan":
        v[rng.integers(m)] = np.nan
    elif kind == "neg_nan":
        v[rng.integers(m)] = np.array(0xFFF8000000000000, np.uint64).view(F64)
    elif kind == "neg_inf":
        v[rng.integers(m)] = -np.inf
    return v


@pytest.mark.parametrize("dtype", [F32, F64], ids=["float32", "float64"])
@pytest.mark.parametrize("kind", KINDS)
def test_threshold_equals_numpy_for_every_small_size(kind, dtype):
    rng = np.random.default_rng([KINDS.index(kind), np.dtype(dtype).itemsize])
    # every size for finite data (the index arithmetic); every size to 256 and then every 13th for the others
    sizes = range(1, 4097) if kind == "finite" else [*range(1, 257), *range(257, 4097, 13), 4096]
    for m in sizes:
        v = _values(rng, m, dtype, kind)
        s = radix_order(v)
        for q in (Q_FINE if m <= 64 or m % 127 == 0 else Q_COARSE):
            got, want = device_threshold(v, q, s), numpy_threshold(v, q)
            assert same(got, want), f"m={m} q={q}: restatement {got!r}, np.percentile {want!r}"


def test_neg_nan_sorts_first_and_nan_last():
    neg_nan = np.array(0xFFF8000000000000, np.uint64).view(F64)
    s = radix_order(np.array([1.0, np.nan, -np.inf, neg_nan, -0.0, 0.0, np.inf, -1.0]))
    assert np.isnan(s[0]) and np.signbit(s[0]) and np.isnan(s[-1]) and not np.signbit(s[-1])
    np.testing.assert_array_equal(s[1:-1], [-np.inf, -1.0, -0.0, 0.0, 1.0, np.inf])
    assert np.signbit(s[3]) and not np.signbit(s[4])


def test_infinite_order_statistics_give_nan():
    # numpy's _lerp: inf - inf is NaN, and so is inf * 0 when the virtual index is an integer below an infinity
    v = np.array([0, 1, 2, np.inf], F32)
    assert np.isnan(numpy_threshold(v, 100.0)) and np.isnan(device_threshold(v, 100.0))
    w = np.array([0, 1, 2, 3, np.inf], F64)
    assert np.isnan(numpy_threshold(w, 75.0)) and np.isnan(device_threshold(w, 75.0))


@pytest.mark.parametrize("m", [2**24 - 1, 2**24, 2**24 + 1, 2**24 + 3, 2**24 + 5, 3 * 2**23 + 1])
def test_float32_threshold_equals_numpy_around_2_24_values(m):
    # non-decreasing non-negative float32 values are already in radix order, so the restatement reads them in place
    rng = np.random.default_rng(m)
    s = np.cumsum(rng.uniform(0.0, 2.0, m)).astype(F32)
    assert (np.diff(s) >= 0).all()
    for q in (0.0, 1e-5, 25.0, 37.5, 50.0, 90.0, 99.99999, 100.0):
        got, want = device_threshold(s, q, s), numpy_threshold(s, q)
        assert same(got, want), f"m={m} q={q}: restatement {got!r}, np.percentile {want!r}"


def test_host_column_sums_are_float32_sums_in_row_order():
    rng = np.random.default_rng(5)
    n = 3000
    rows = np.concatenate([np.arange(n), rng.integers(0, n, 200_000)])
    cols = np.concatenate([np.zeros(n, np.int64), rng.integers(0, 40, 200_000)])  # a star column and 40 columns of high in-degree
    a = sp.csr_matrix((rng.uniform(0.1, 1.0, rows.size).astype(F32), (rows, cols)), shape=(n, n))
    a.sum_duplicates()
    got = np.asarray(a.sum(axis=0)).ravel()
    assert got.dtype == F32
    want = np.zeros(n, F32)
    np.add.at(want, a.indices, a.data)  # every column from 0, one float32 entry after another, rows ascending
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    f64 = np.asarray(a.sum(axis=0, dtype=F64)).ravel().astype(F32)
    assert (f64 != want).any(), "the float64 column sums rounded to float32 should differ from the float32 sums in some column"
