"""Known answers for Moran's I / Geary's C that do not come from this repository's own restatement.

The reference delegates the arithmetic to ``scanpy.metrics.morans_i / gearys_c`` (``src/squidpy/gr/_ppatterns.py:216``),
which cannot be imported here, and no reference test pins a numeric I or C.  What CAN be pinned is the published
definition the reference documents (``_ppatterns.py:76-150``; variance code ``:501-538``):

    I = N/S0 * sum_ij w_ij z_i z_j / sum_i z_i^2          z = x - mean(x),  S0 = sum_ij w_ij  (W as given, NOT symmetrised)
    C = (N-1) * sum_ij w_ij (x_i - x_j)^2 / (2 * S0 * sum_i z_i^2)

Two independent sources of truth are used:
  * closed forms derived by hand for structured fields (the derivations are in the comments of ``CASES``; the expected
    values are literals);
  * :func:`exact_autocorr` — the definition evaluated in exact rational arithmetic (``fractions.Fraction``; float32 /
    float64 inputs are exact rationals), i.e. the value every correct floating-point implementation must round to.
What stays unpinned after this: only scanpy's floating-point operation ORDER (last-bit differences).
"""

from __future__ import annotations

from fractions import Fraction

import numpy as np
import scipy.sparse as sp


def exact_autocorr(w: sp.spmatrix, x: np.ndarray) -> tuple[float, float]:
    """(I, C) of one feature by exact rational arithmetic over the stored entries of ``w`` (duplicates kept)."""
    w = sp.csr_matrix(w)
    n = w.shape[0]
    xs = [Fraction(float(v)) for v in np.asarray(x).ravel()]
    mean = sum(xs, Fraction(0)) / n
    z = [v - mean for v in xs]
    z2 = sum((v * v for v in z), Fraction(0))
    s0 = Fraction(0)
    num_i = Fraction(0)
    num_c = Fraction(0)
    for i in range(n):
        for e in range(w.indptr[i], w.indptr[i + 1]):
            j = int(w.indices[e])
            wij = Fraction(float(w.data[e]))
            s0 += wij
            num_i += wij * z[i] * z[j]
            num_c += wij * (xs[i] - xs[j]) ** 2
    if z2 == 0:
        return float("nan"), float("nan")
    return float(Fraction(n) / s0 * num_i / z2), float(Fraction(n - 1) * num_c / (2 * s0 * z2))


def torus_grid(side: int, dtype=np.float32, normalise: bool = False) -> sp.csr_matrix:
    """4-neighbour periodic square grid, node (r, c) -> r*side + c."""
    rows, cols = [], []
    for r in range(side):
        for c in range(side):
            for dr, dc in ((1, 0), (-1, 0), (0, 1), (0, -1)):
                rows.append(r * side + c)
                cols.append(((r + dr) % side) * side + (c + dc) % side)
    g = sp.csr_matrix((np.ones(len(rows), dtype), (rows, cols)), shape=(side * side, side * side))
    g.sort_indices()
    if normalise:
        g.data[:] = dtype(0.25)  # 1/4 is exact in binary floating point
    return g


def path_graph(n: int, dtype=np.float32) -> sp.csr_matrix:
    i = np.arange(n - 1)
    g = sp.csr_matrix((np.ones(2 * (n - 1), dtype), (np.r_[i, i + 1], np.r_[i + 1, i])), shape=(n, n))
    g.sort_indices()
    return g


def five_node_asymmetric() -> tuple[sp.csr_matrix, np.ndarray]:
    """Directed 5-node graph, float32 weights row-normalised IN float32 (what ``transformation=True`` produces,
    ``_ppatterns.py:212-214``): row 0 -> {1, 2, 3} (1/3 each as float32), row 1 -> {0}, row 2 -> {1, 4} (weights 0.25 and
    0.75), row 3 -> {} (isolated source), row 4 -> {0, 1, 2, 3} (0.25 each).  W is NOT symmetric: pins 'S0 = sum(W.data),
    W used as given'."""
    third = np.float32(1.0) / np.float32(3.0)
    rows = [0, 0, 0, 1, 2, 2, 4, 4, 4, 4]
    cols = [1, 2, 3, 0, 1, 4, 0, 1, 2, 3]
    data = np.array([third, third, third, 1.0, 0.25, 0.75, 0.25, 0.25, 0.25, 0.25], dtype=np.float32)
    g = sp.csr_matrix((data, (rows, cols)), shape=(5, 5))
    g.sort_indices()
    x = np.array([1.0, 0.0, 2.5, 0.0, -1.5], dtype=np.float32)
    return g, x


def _cases():
    out = []
    # 1. checkerboard x = (-1)^(r+c) on a 6x6 torus, binary weights: mean 0, every neighbour has the opposite sign, so
    #    sum_ij w_ij z_i z_j = -4N, S0 = 4N, sum z^2 = N  =>  I = N/(4N) * (-4N)/N = -1 exactly;
    #    sum_ij w_ij (x_i-x_j)^2 = 4N * 4  =>  C = (N-1) * 16N / (2 * 4N * N) = 2(N-1)/N = 70/36.
    side = 6
    rc = np.add.outer(np.arange(side), np.arange(side)).ravel()
    chk = np.where(rc % 2 == 0, 1.0, -1.0)
    out.append(("checkerboard_torus_binary", torus_grid(side), chk, -1.0, 70.0 / 36.0))
    # 2. the same field with row-normalised weights (1/4 each): S0 = N, numerator = -N  =>  I = -1;  C numerator = 4N,
    #    C = (N-1) * 4N / (2 * N * N) = 2(N-1)/N again.
    out.append(("checkerboard_torus_rownorm", torus_grid(side, normalise=True), chk, -1.0, 70.0 / 36.0))
    # 3. two blocks on a path graph of n = 10 nodes, x = 1 on the first half, 0 on the second: z = +-1/2, sum z^2 = n/4;
    #    directed edges: 2(n-2) with equal signs (+1/4 each), 2 across the boundary (-1/4 each) => num = (n-3)/2;
    #    S0 = 2(n-1)  =>  I = n/(2(n-1)) * ((n-3)/2) / (n/4) = (n-3)/(n-1) = 7/9;
    #    sum w (x_i-x_j)^2 = 2  =>  C = (n-1) * 2 / (2 * 2(n-1) * n/4) = 2/n = 0.2.
    n = 10
    blocks = np.r_[np.ones(n // 2), np.zeros(n // 2)]
    out.append(("two_blocks_path", path_graph(n), blocks, 7.0 / 9.0, 0.2))
    # 4. linear gradient x_i = i on the same path graph: sum z^2 = n(n^2-1)/12; z_i z_{i+1} = z_i^2 + z_i and
    #    sum_{i<n-1} (z_i^2 + z_i) = (n-1)(n-3)(n+1)/12  =>  I = n/(2(n-1)) * 2(n-1)(n-3)(n+1)/12 / (n(n^2-1)/12)
    #    = (n-3)/(n-1) = 7/9;   sum w (x_i-x_j)^2 = 2(n-1)  =>  C = (n-1) * 2(n-1) / (2 * 2(n-1) * n(n^2-1)/12)
    #    = 6/(n(n+1)) = 6/110.
    out.append(("gradient_path", path_graph(n), np.arange(n, dtype=np.float64), 7.0 / 9.0, 6.0 / 110.0))
    # 5. asymmetric float32 row-normalised W on 5 nodes: literals = exact rational evaluation of the definition with the
    #    float32 weights as stored (1/3 -> 0x3EAAAAAB), rounded to float64 (tests re-derive them with exact_autocorr).
    g5, x5 = five_node_asymmetric()
    out.append(("five_node_asymmetric_f32", g5, x5, FIVE_NODE_I, FIVE_NODE_C))
    return out


# exact values of case 5 (see tests/test_autocorr_known_answers.py::test_five_node_literals_are_exact)
FIVE_NODE_I = -0.5869252818700825
FIVE_NODE_C = 1.302681985057862

CASES = _cases()


def dense_longdouble(w: sp.spmatrix, x: np.ndarray) -> tuple[float, float]:
    """Third formulation: dense matrix algebra in ``np.longdouble`` (x87 80-bit here), z'Wz / z'z — shares no loop
    structure with the CSR restatement or the CUDA kernels."""
    wd = np.asarray(sp.csr_matrix(w).todense(), dtype=np.longdouble)
    xl = np.asarray(x, dtype=np.longdouble)
    n = xl.size
    z = xl - xl.sum() / n
    s0 = wd.sum()
    z2 = (z * z).sum()
    diff = xl[:, None] - xl[None, :]
    return float(n / s0 * (z @ (wd @ z)) / z2), float((n - 1) * (wd * diff * diff).sum() / (2 * s0 * z2))


def _longdouble_terms(w: sp.spmatrix, x: np.ndarray):
    """W's stored entries (rows, cols, weights) and the centred feature, all in ``np.longdouble``.  The mean is kept as
    two parts, ``mean + low`` with ``low`` the mean of the residuals: a single long double holds a mean of 1e6 only to
    ~1e-13, which would shift every z by that much; with the second part z is accurate to its own long-double epsilon."""
    w = sp.csr_matrix(w)
    n = w.shape[0]
    xl = np.asarray(x, dtype=np.longdouble).ravel()
    mean = xl.sum() / n
    low = (xl - mean).sum() / n
    rows = np.repeat(np.arange(n), np.diff(w.indptr))
    return w, rows, w.indices, w.data.astype(np.longdouble), xl, mean, (xl - mean) - low


def sparse_longdouble(w: sp.spmatrix, x: np.ndarray) -> tuple[float, float]:
    """(I, C) of one feature: the definition over the stored entries of ``w`` in ``np.longdouble``, never densified (N = 1M
    takes about a second).  ``(Wz)_i`` is summed per row; Geary's numerator comes straight from the differences
    ``x_i - x_j``.  A constant feature (every value equal, compared exactly) is the definition's 0/0: NaN."""
    w, rows, cols, wd, xl, _, z = _longdouble_terms(w, x)
    n = w.shape[0]
    if xl.min() == xl.max():
        return float("nan"), float("nan")
    s0 = wd.sum()
    z2 = (z * z).sum()
    wz = np.zeros(n, dtype=np.longdouble)
    full = np.diff(w.indptr) > 0
    if w.nnz:
        wz[full] = np.add.reduceat(wd * z[cols], w.indptr[:-1][full])
    diff = xl[rows] - xl[cols]
    return float(n / s0 * (z * wz).sum() / z2), float((n - 1) * (wd * diff * diff).sum() / (2 * s0 * z2))


def autocorr_scale(w: sp.spmatrix, x: np.ndarray) -> tuple[float, float]:
    """First-order error scale of a float64 evaluation of (I, C): the sum of |partial derivative| x |operand| over the
    rounded operations, so that a careful evaluation is off by a modest multiple of eps x scale.  A test bounds
    ``|got - ref| <= k * scale`` where I or C is near 0 and a relative bound means nothing.

    I: ``(N/S0) * (sum |w_ij||z_i||z_j| + |m| * |sum_ij w_ij (z_i + z_j)|) / sum z^2``.  The first term covers the rounding of
    every product and partial sum.  The second covers the mean: ``sum x / N`` in float64 is off by about eps * |m|, which
    shifts every z by the same amount and moves ``z'Wz`` by that shift times ``sum_ij w_ij (z_i + z_j)``; ``sum z^2`` moves
    only at second order.  Without it no float64 evaluation could meet the bound once |m| >> std(x).
    C: ``(N-1) * sum |w_ij| (x_i - x_j)^2 / (2 * S0 * sum z^2)``; the differences do not involve the mean, and for
    non-negative weights this is C itself."""
    w, rows, cols, wd, xl, mean, z = _longdouble_terms(w, x)
    n = w.shape[0]
    s0 = wd.sum()
    z2 = (z * z).sum()
    aw = np.abs(wd)
    si = (aw * np.abs(z[rows]) * np.abs(z[cols])).sum() + abs(mean) * abs((wd * (z[rows] + z[cols])).sum())
    diff = xl[rows] - xl[cols]
    return float(n / abs(s0) * si / z2), float((n - 1) * (aw * diff * diff).sum() / (2 * abs(s0) * z2))
