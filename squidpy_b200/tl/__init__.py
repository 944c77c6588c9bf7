"""``squidpy_b200.tl`` — ``squidpy.tl`` tools whose cost is a spatial search, on an H100."""

from ._sliding_window import _calculate_window_corners, sliding_window, window_ranges
from ._var_by_distance import nn_min_dist, var_by_distance

__all__ = ["sliding_window", "var_by_distance", "nn_min_dist", "window_ranges"]
