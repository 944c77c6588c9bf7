"""Executable specification of the device build of spatial_autocorr's weight matrix W (``sqb_autocorr_create_device``): the
l1 row normalisation of ``sklearn.preprocessing.normalize``, numpy's pairwise summation, the moments s0 / s1 / s2 of
``_g_moments`` (scipy's operation order for a canonical CSR, in W's dtype) and the predicate under which S0 is summed exactly
in parallel.  The CPU tests pin every function here to the library it restates; the kernels follow it step for step."""

from __future__ import annotations

import numpy as np

PW_BLOCK = 128  # numpy's PW_BLOCKSIZE


def l1_normalize(indptr: np.ndarray, data: np.ndarray) -> np.ndarray:
    """``normalize(W, norm="l1", axis=1)`` of a float32 / float64 CSR: per row a sequential float64 sum of |w| in entry
    order; rows whose sum is 0 are left as they are; every value becomes ``(T)((double)w / sum)``."""
    out = data.copy()
    for r in range(indptr.size - 1):
        a, b = int(indptr[r]), int(indptr[r + 1])
        s = 0.0
        for e in range(a, b):
            s += abs(float(data[e]))
        if s != 0.0:
            out[a:b] = (data[a:b].astype(np.float64) / s).astype(data.dtype)
    return out


def _leaf(a: np.ndarray) -> np.generic:
    """numpy's pairwise_sum for n <= 128: a plain loop below 8, else eight strided accumulators and the tail in order."""
    t = a.dtype.type
    n = a.size
    if n < 8:
        r = t(0.0)
        for v in a:
            r = t(r + v)
        return r
    m = n - n % 8
    r = list(a[:8])
    for i in range(8, m, 8):
        for j in range(8):
            r[j] = t(r[j] + a[i + j])
    res = t(t(t(r[0] + r[1]) + t(r[2] + r[3])) + t(t(r[4] + r[5]) + t(r[6] + r[7])))
    for v in a[m:]:
        res = t(res + v)
    return res


def pairwise(a: np.ndarray) -> np.generic:
    """numpy's pairwise summation of a contiguous float array in its own dtype (the zero it starts from aside)."""
    n = a.size
    if n <= PW_BLOCK:
        return _leaf(a)
    n2 = n // 2
    n2 -= n2 % 8
    return a.dtype.type(pairwise(a[:n2]) + pairwise(a[n2:]))


def np_sum(a: np.ndarray) -> np.generic:
    """``np.sum`` of a contiguous float32 / float64 array: +0.0 plus the pairwise sum."""
    return a.dtype.type(a.dtype.type(0.0) + pairwise(a))


def row_sums(indptr: np.ndarray, data: np.ndarray) -> np.ndarray:
    """``W.sum(1)`` of a CSR (``np.add.reduceat`` over the non-empty rows): the row's first value plus the pairwise sum of
    the rest; 0 for an empty row."""
    t = data.dtype.type
    out = np.zeros(indptr.size - 1, data.dtype)
    for r in range(indptr.size - 1):
        a, b = int(indptr[r]), int(indptr[r + 1])
        if b > a:
            out[r] = t(data[a] + pairwise(data[a + 1 : b])) if b - a > 1 else data[a]
    return out


def col_sums(n: int, indices: np.ndarray, data: np.ndarray) -> np.ndarray:
    """``W.sum(0)`` (a product with ones): a sequential sum per column in entry (row) order, from 0."""
    out = np.zeros(n, data.dtype)
    np.add.at(out, indices, data)
    return out


def sym_values(n: int, indptr: np.ndarray, indices: np.ndarray, data: np.ndarray) -> np.ndarray:
    """The stored values of ``W.T + W`` for a canonical CSR W: w_ij + w_ji in W's dtype, zeros dropped, in row-major order
    (scipy returns a canonical CSC; the matrix is symmetric, so its column-major order is this row-major order)."""
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(indptr))
    cols = indices.astype(np.int64)
    i = np.concatenate([rows, cols])
    j = np.concatenate([cols, rows])
    v = np.concatenate([data, data])
    order = np.lexsort((j, i))
    i, j, v = i[order], j[order], v[order]
    key = i * n + j
    first = np.ones(key.size, bool)
    first[1:] = key[1:] != key[:-1]
    starts = np.flatnonzero(first)
    t = v[starts].copy()
    pair = np.zeros(key.size, bool)
    pair[:-1] = ~first[1:]  # an entry whose successor has the same (i, j): at most two per key
    two = pair[starts]
    t[two] = (v[starts[two]] + v[starts[two] + 1]).astype(data.dtype)
    return t[t != 0]


def g_moments(n: int, indptr: np.ndarray, indices: np.ndarray, data: np.ndarray) -> tuple:
    """s0, s1, s2 of ``_g_moments`` for a canonical CSR W (float32 or float64), as the same numpy scalar types."""
    t = data.dtype.type
    s0 = np_sum(data)
    sym = sym_values(n, indptr, indices, data)
    sq = (sym * sym).astype(data.dtype)
    s1 = t(np_sum(sq[sq != 0]) / 2.0)
    rc = (row_sums(indptr, data) + col_sums(n, indices, data)).astype(data.dtype)
    s2 = np_sum((rc * rc).astype(data.dtype))
    return s0, s1, s2


def lowest_bit_exponent(w: np.ndarray) -> np.ndarray:
    """e with 2**e the lowest set bit of every non-zero finite float64 value (its smallest ulp multiple)."""
    m, e = np.frexp(w)  # w = m * 2**e, 0.5 <= |m| < 1: the 53-bit significand is m * 2**53
    sig = np.abs(m * 2.0**53).astype(np.int64)
    tz = np.zeros(sig.size, np.int64)
    s = sig.copy()
    while np.any((s & 1) == 0):
        z = (s & 1) == 0
        tz[z] += 1
        s[z] >>= 1
    return e.astype(np.int64) - 53 + tz


def s0_exact_predicate(wd: np.ndarray) -> bool:
    """True when the sequential float64 sum of ``wd`` (float64 weights) is exact, hence equal to the integer sum of w / g:
    every weight is a multiple of g = the smallest lowest set bit among them, and sum |w| < 2**53 g keeps every partial sum
    a representable multiple of g.  Non-finite weights fail it."""
    if not np.all(np.isfinite(wd)):
        return False
    nz = wd[wd != 0]
    if nz.size == 0:
        return True
    g = int(lowest_bit_exponent(nz).min())
    return bool(np.sum(np.abs(nz)) < np.ldexp(1.0, 53 + g))


def s0_sequential(wd: np.ndarray) -> float:
    s = 0.0
    for v in wd:
        s += float(v)
    return s


def s0_exact(wd: np.ndarray) -> float:
    """The integer-sum form of S0 (valid under ``s0_exact_predicate``)."""
    nz = wd[wd != 0]
    if nz.size == 0:
        return 0.0
    g = int(lowest_bit_exponent(nz).min())
    k = sum(int(v) for v in np.ldexp(nz, -g).astype(np.int64))
    return float(np.ldexp(float(k), g))
