"""Graph construction strategies for spatial neighbour graphs: the public names of ``squidpy.gr.neighbors``
(``src/squidpy/gr/neighbors.py:33-45``).  Subclass :class:`GraphBuilderCSR` and pass an instance to
:func:`~squidpy_b200.gr.spatial_neighbors_from_builder` to build a custom graph; the built-in builders are the ones
``squidpy_b200.gr`` exports."""

from ._build import DelaunayBuilder, GridBuilder, KNNBuilder, RadiusBuilder
from ._postprocess import (DistanceIntervalPostprocessor, GraphBuilder, GraphBuilderCSR, GraphMatrixT, GraphPostprocessor, PercentilePostprocessor,
                           TransformPostprocessor)

__all__ = [
    "GraphMatrixT",
    "GraphBuilder",
    "GraphBuilderCSR",
    "GraphPostprocessor",
    "DistanceIntervalPostprocessor",
    "PercentilePostprocessor",
    "TransformPostprocessor",
    "KNNBuilder",
    "RadiusBuilder",
    "DelaunayBuilder",
    "GridBuilder",
]
