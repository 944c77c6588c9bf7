"""CPU restatement of ``sqb_nn_dist_hist_f64`` (test infrastructure): nearest-neighbour distance histograms from
scikit-learn's ``KDTree.query`` and ``np.histogram``, and the kernel's binning on squared distances."""

from __future__ import annotations

import numpy as np


def nn_dist_hist(ref_pts: np.ndarray, qry_pts: np.ndarray, k: int, support: np.ndarray) -> np.ndarray:
    """``np.histogram`` of the k nearest distances of every query point among ``ref_pts`` (kd_tree arithmetic: float64
    ``sqrt(dx*dx + dy*dy)``, no point excluded): int64 (len(support) - 1,)."""
    from sklearn.neighbors import KDTree

    support = np.asarray(support, dtype=np.float64)
    qry = np.asarray(qry_pts, dtype=np.float64).reshape(-1, 2)
    if qry.shape[0] == 0:
        return np.zeros(support.size - 1, dtype=np.int64)
    d, _ = KDTree(np.asarray(ref_pts, dtype=np.float64).reshape(-1, 2)).query(qry, k=k)
    return np.histogram(d.ravel(), bins=support)[0].astype(np.int64)


def eval_tasks(points: np.ndarray, tasks: np.ndarray, support: np.ndarray, n_rows: int) -> np.ndarray:
    """``nn_distance_hist`` evaluated on the host: every task (ref_begin, ref_end, qry_begin, qry_end, k, row) with
    :func:`nn_dist_hist`, summed per row."""
    out = np.zeros((n_rows, len(support) - 1), dtype=np.int64)
    for rb, re, qb, qe, k, row in np.asarray(tasks, dtype=np.int64).reshape(-1, 6):
        out[row] += nn_dist_hist(points[rb:re], points[qb:qe], int(k), support)
    return out


def d2_thresholds(support: np.ndarray) -> np.ndarray:
    """The kernel's thresholds: thr[j] = min{t >= 0 : sqrt(t) >= e[j]} for j < S - 1, thr[S - 1] = max{t : sqrt(t) <= e[S - 1]}."""
    e = np.asarray(support, dtype=np.float64)
    thr = np.empty(e.size)
    for j, r in enumerate(e[:-1]):
        if r <= 0 or np.isinf(r):
            thr[j] = 0.0 if r <= 0 else np.inf
            continue
        t = r * r
        while np.sqrt(t) < r:
            t = np.nextafter(t, np.inf)
        while t > 0 and np.sqrt(np.nextafter(t, 0.0)) >= r:
            t = np.nextafter(t, 0.0)
        thr[j] = t
    r = e[-1]
    if r < 0 or np.isinf(r):
        thr[-1] = -1.0 if r < 0 else np.inf
    else:
        t = r * r
        while np.sqrt(t) > r:
            t = np.nextafter(t, 0.0)
        while np.isfinite(np.nextafter(t, np.inf)) and np.sqrt(np.nextafter(t, np.inf)) <= r:
            t = np.nextafter(t, np.inf)
        thr[-1] = t
    return thr


def bin_d2(d2: np.ndarray, support: np.ndarray) -> np.ndarray:
    """The kernel's binning (``nnd_bin``) of squared distances: bin i = #{j < S - 1 : thr[j] <= d2} - 1 when
    thr[0] <= d2 <= thr[S - 1], else dropped.  Returns the int64 histogram."""
    thr = d2_thresholds(support)
    d2 = np.asarray(d2, dtype=np.float64).ravel()
    keep = (d2 >= thr[0]) & (d2 <= thr[-1])
    b = np.searchsorted(thr[:-1], d2[keep], side="right") - 1
    return np.bincount(b, minlength=len(support) - 1).astype(np.int64)
