"""Kernel codes of scikit-learn's metric names, shared by every entry point that takes a ``KDTree`` metric
(``sqb_pair_counts_f64``, ``sqb_nn_min_dist_f64``)."""

from __future__ import annotations

import numpy as np

__all__ = ["metric_code"]

_METRIC_CODES = {"EuclideanDistance": 0, "ManhattanDistance": 1, "ChebyshevDistance": 2}


def metric_code(metric: str) -> int:
    """Kernel code of a metric name: 0 euclidean, 1 manhattan, 2 chebyshev, the classes ``DistanceMetric.get_metric`` resolves
    every ``KDTree`` metric name to.  Names it rejects raise its error; metrics ``KDTree`` does not take raise KDTree's."""
    from sklearn.metrics import DistanceMetric
    from sklearn.neighbors import KDTree

    dm = DistanceMetric.get_metric(metric)
    name = type(dm).__name__.rstrip("0123456789")
    if name not in _METRIC_CODES:
        KDTree(np.zeros((1, 2)), metric=dm)  # ValueError: not valid for KDTree
        raise NotImplementedError(f"the GPU kernels have no distance for the metric `{metric}`.")
    return _METRIC_CODES[name]
