"""Pure-Python restatement of the per-point star construction of ``csrc/delaunay.cu`` with exact rational predicates: the
same ghost rule, the same symbolic perturbation of x^2 + y^2 by index and the same duplicate rule (lowest index of a group is
the vertex, the other copies get empty rows).  Every point is offered every other distinct point, so the result does not
depend on the grid or on the passes.  Slow (O(n^2) predicates): for inputs of a few hundred points."""

from __future__ import annotations

from fractions import Fraction as F

import numpy as np

GHOST = -1


def _sgn(x):
    return (x > 0) - (x < 0)


def orient(a, b, c):
    return _sgn((a[0] - c[0]) * (b[1] - c[1]) - (a[1] - c[1]) * (b[0] - c[0]))


def incircle(a, b, c, d):
    rows = [(p[0] - d[0], p[1] - d[1]) for p in (a, b, c)]
    (a1, a2), (b1, b2), (c1, c2) = rows
    a3, b3, c3 = a1 * a1 + a2 * a2, b1 * b1 + b2 * b2, c1 * c1 + c2 * c2
    return _sgn(a1 * (b2 * c3 - b3 * c2) - a2 * (b1 * c3 - b3 * c1) + a3 * (b1 * c2 - b2 * c1))


def incircle_sos(a, b, c, d, ia, ib, ic, id_):
    s = incircle(a, b, c, d)
    if s:
        return s
    coef = {ia: orient(d, b, c), ib: orient(d, c, a), ic: orient(d, a, b), id_: -orient(a, b, c)}
    for k in sorted(coef, reverse=True):
        if coef[k]:
            return coef[k]
    return 0


def _between(a, b, l):
    if a[0] != b[0]:
        return min(a[0], b[0]) < l[0] < max(a[0], b[0])
    return min(a[1], b[1]) < l[1] < max(a[1], b[1])


def _conflicts(P, i, p, q, l):
    if l in (p, q):
        return False
    if p == GHOST:
        o = orient(P[i], P[l], P[q])
        return o > 0 or (o == 0 and _between(P[i], P[q], P[l]))
    if q == GHOST:
        o = orient(P[i], P[p], P[l])
        return o > 0 or (o == 0 and _between(P[i], P[p], P[l]))
    return incircle_sos(P[i], P[p], P[q], P[l], i, p, q, l) > 0


def star_insert(P, i, s, l):
    m = len(s)
    c = [_conflicts(P, i, s[k], s[(k + 1) % m], l) for k in range(m)]
    if not any(c):
        return s
    if all(c):
        raise AssertionError("every triangle of the star conflicts")
    start = next(k for k in range(m) if c[k] and not c[k - 1])
    end = next(k for k in range(m) if c[k] and not c[(k + 1) % m])
    keep = [s[(end + 1 + t) % m] for t in range(m - (end - start) % m)]
    return keep + [l]


def delaunay_rows(xy) -> tuple[np.ndarray, np.ndarray]:
    """(indptr, indices) of the Delaunay graph, rows ascending; raises ValueError for < 3 distinct or collinear points."""
    xy = np.asarray(xy, dtype=np.float64)
    n = xy.shape[0]
    P = [(F(float(x)), F(float(y))) for x, y in xy]
    rep = {}
    reps = []
    for k, p in enumerate(P):
        rep.setdefault(p, k)
        if rep[p] == k:
            reps.append(k)
    rows = [[] for _ in range(n)]
    for i in reps:
        order = sorted((j for j in reps if j != i), key=lambda j: ((P[j][0] - P[i][0]) ** 2 + (P[j][1] - P[i][1]) ** 2, j))
        if not order:
            raise ValueError("fewer than three distinct points")
        a = order[0]
        b = next((j for j in order if orient(P[i], P[a], P[j]) != 0), None)
        if b is None:
            raise ValueError("all points collinear")
        s = [a, b, GHOST] if orient(P[i], P[a], P[b]) > 0 else [b, a, GHOST]
        for l in order:
            if l not in (a, b):
                s = star_insert(P, i, s, l)
        rows[i] = sorted(v for v in s if v != GHOST)
    indptr = np.zeros(n + 1, dtype=np.int64)
    indptr[1:] = np.cumsum([len(r) for r in rows])
    return indptr, np.array([v for r in rows for v in r], dtype=np.int32)
