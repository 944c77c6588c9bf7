"""CPU restatement of ``sqb_pair_counts_f64`` for every metric code (test infrastructure): brute force in numpy with the
arithmetic of scikit-learn's ``KDTree(p, metric=...).two_point_correlation(p, support)``, whose ``_two_point_dual`` counts the
ordered pairs, self pairs included, with ``dist(p, q) <= r`` (the tree only prunes; the integers are the same)."""

from __future__ import annotations

import numpy as np

METRICS = {0: "euclidean", 1: "manhattan", 2: "chebyshev"}
NAMES = {0: ["euclidean", "l2", "minkowski", "p"], 1: ["manhattan", "cityblock", "l1"], 2: ["chebyshev", "infinity"]}


def pair_dist(dx: np.ndarray, dy: np.ndarray, metric: int) -> np.ndarray:
    """sqrt(dx*dx + dy*dy) (numpy never contracts to an FMA) / |dx| + |dy| / max(|dx|, |dy|), float64."""
    if metric == 0:
        return np.sqrt(dx * dx + dy * dy)
    if metric == 1:
        return np.abs(dx) + np.abs(dy)
    if metric == 2:
        return np.maximum(np.abs(dx), np.abs(dy))
    raise ValueError(metric)


def pair_counts(points: np.ndarray, support: np.ndarray, metric: int) -> np.ndarray:
    """int64 (S,): #{ordered (i, j), i == j included : dist(p_i, p_j) <= support[s]}."""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 2)
    sup = np.asarray(support, dtype=np.float64)
    out = np.zeros(sup.size, dtype=np.int64)
    for s in range(0, p.shape[0], 1024):
        d = np.sort(pair_dist(p[s : s + 1024, None, 0] - p[None, :, 0], p[s : s + 1024, None, 1] - p[None, :, 1], metric), axis=None)
        out += np.searchsorted(d, sup, side="right")  # -0.0 == 0.0 in the comparison, as in `<=`
    return out


def group_counts(groups: list[np.ndarray], support: np.ndarray, metric: int) -> np.ndarray:
    """``pair_counts(groups, support, metric=metric)`` of the library: int64 (len(groups), S)."""
    return np.stack([pair_counts(g, support, metric) for g in groups]).reshape(len(groups), np.asarray(support).size)
