"""CPU restatement of ``sqb_nn_min_dist_f64`` (test infrastructure): every task's nearest-reference distances from
scikit-learn's ``KDTree.query``, and brute force in numpy with the kernel's arithmetic."""

from __future__ import annotations

import numpy as np

METRICS = {0: "euclidean", 1: "manhattan", 2: "chebyshev"}


def brute_min_dist(ref: np.ndarray, qry: np.ndarray, metric: int) -> np.ndarray:
    """min over ref of sqrt(dx*dx + dy*dy) / |dx| + |dy| / max(|dx|, |dy|), float64, for every query point."""
    out = np.empty(qry.shape[0])
    for s in range(0, qry.shape[0], 2048):
        dx = qry[s : s + 2048, None, 0] - ref[None, :, 0]
        dy = qry[s : s + 2048, None, 1] - ref[None, :, 1]
        if metric == 0:
            out[s : s + 2048] = np.sqrt((dx * dx + dy * dy).min(axis=1))
        elif metric == 1:
            out[s : s + 2048] = (np.abs(dx) + np.abs(dy)).min(axis=1)
        else:
            out[s : s + 2048] = np.maximum(np.abs(dx), np.abs(dy)).min(axis=1)
    return out


def eval_tasks(points: np.ndarray, tasks: np.ndarray, metric: int, n_out: int) -> np.ndarray:
    """``nn_min_dist`` evaluated on the host with ``KDTree(ref, metric=DistanceMetric.get_metric(m)).query(qry)``."""
    from sklearn.metrics import DistanceMetric
    from sklearn.neighbors import KDTree

    points = np.asarray(points, dtype=np.float64).reshape(-1, 2)
    out = np.full(int(n_out), np.nan)
    for rb, re, qb, qe, ob in np.asarray(tasks, dtype=np.int64).reshape(-1, 5):
        if qe > qb:
            d, _ = KDTree(points[rb:re], metric=DistanceMetric.get_metric(METRICS[int(metric)])).query(points[qb:qe])
            out[ob : ob + (qe - qb)] = d[:, 0]
    return out
