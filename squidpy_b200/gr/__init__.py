"""``squidpy_b200.gr`` — the spatial-statistics hot path of ``squidpy.gr`` on an H100."""

from ._build import (DelaunayBuilder, GridBuilder, KNNBuilder, RadiusBuilder, SpatialNeighborsResult, delaunay_2d, knn_2d, radius_2d,
                     spatial_neighbors, spatial_neighbors_delaunay, spatial_neighbors_from_builder, spatial_neighbors_grid, spatial_neighbors_knn,
                     spatial_neighbors_radius)
from . import neighbors
from ._mask import mask_graph
from ._ligrec import ligrec, ligrec_analysis, ligrec_analysis_device
from ._niche import (calculate_niche, calculate_niche_cellcharter, calculate_niche_neighborhood, calculate_niche_spatialleiden,
                     calculate_niche_utag, niche_aggregate, niche_profile)
from ._nhood import NhoodEnrichmentResult, NhoodPlan, centrality_counts, centrality_scores, interaction_matrix, nhood_enrichment
from ._ppatterns import AutocorrPlan, co_occurrence, cooc_counts, spatial_autocorr
from ._ripley import nn_distance_hist, pair_counts, ripley
from ._sepal import sepal, sepal_scores

__all__ = [
    "spatial_neighbors",
    "spatial_neighbors_knn",
    "spatial_neighbors_grid",
    "spatial_neighbors_radius",
    "spatial_neighbors_delaunay",
    "spatial_neighbors_from_builder",
    "mask_graph",
    "SpatialNeighborsResult",
    "DelaunayBuilder",
    "delaunay_2d",
    "KNNBuilder",
    "GridBuilder",
    "RadiusBuilder",
    "knn_2d",
    "radius_2d",
    "ligrec",
    "sepal",
    "sepal_scores",
    "ligrec_analysis",
    "ligrec_analysis_device",
    "nhood_enrichment",
    "interaction_matrix",
    "centrality_scores",
    "centrality_counts",
    "calculate_niche",
    "calculate_niche_neighborhood",
    "calculate_niche_utag",
    "calculate_niche_cellcharter",
    "calculate_niche_spatialleiden",
    "niche_profile",
    "niche_aggregate",
    "spatial_autocorr",
    "co_occurrence",
    "ripley",
    "NhoodEnrichmentResult",
    "NhoodPlan",
    "AutocorrPlan",
    "cooc_counts",
    "pair_counts",
    "nn_distance_hist",
]
