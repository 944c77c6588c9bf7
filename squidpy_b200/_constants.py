"""Key strings and mode enums of the hot path (contract with AnnData and ``sq.pl``).

Mirrors ``src/squidpy/_constants/_pkg_constants.py:65-121,198-213`` (``Key``) and
``src/squidpy/_constants/_constants.py:74-77,93-110`` (``Centrality``, ``SpatialAutocorr``, ``RipleyStat``) of the reference, including the
error text of an invalid enum value (``_constants/_utils.py:30-40``).
"""

from __future__ import annotations

from enum import Enum, unique


class ModeEnum(str, Enum):
    """String enum that lists the valid options when an invalid value is passed."""

    @classmethod
    def _missing_(cls, value):
        raise ValueError(
            f"Invalid option `{value}` for `{cls.__name__}`. Valid options are: `{[m.value for m in cls]}`."
        )

    @property
    def s(self) -> str:
        return str(self.value)

    @property
    def v(self):
        return self.value

    def __str__(self) -> str:
        return str(self.value)

    __repr__ = __str__


@unique
class SpatialAutocorr(ModeEnum):
    MORAN = "moran"
    GEARY = "geary"


@unique
class Transform(Enum):
    """Adjacency transforms of the graph builders (``_constants/_constants.py:33-36``); ``NONE`` carries the value ``None``."""

    SPECTRAL = "spectral"
    COSINE = "cosine"
    NONE = None

    @classmethod
    def _missing_(cls, value):
        raise ValueError(f"Invalid option `{value}` for `{cls.__name__}`. Valid options are: `{[m.value for m in cls]}`.")

    @property
    def s(self) -> str:
        return str(self.value)

    @property
    def v(self):
        return self.value

    def __str__(self) -> str:
        return str(self.value)


@unique
class CoordType(ModeEnum):
    GRID = "grid"
    GENERIC = "generic"


@unique
class CorrAxis(ModeEnum):
    INTERACTIONS = "interactions"
    CLUSTERS = "clusters"


@unique
class ComplexPolicy(ModeEnum):
    MIN = "min"
    ALL = "all"


@unique
class RipleyStat(ModeEnum):
    F = "F"
    G = "G"
    L = "L"


@unique
class Centrality(ModeEnum):
    DEGREE = "degree_centrality"
    CLUSTERING = "average_clustering"
    CLOSENESS = "closeness_centrality"


class Key:
    class obsm:
        spatial = "spatial"

    class obsp:
        @staticmethod
        def _spatial_key(value: str | None, suffix: str) -> str:
            if value is None:
                return f"{Key.obsm.spatial}_{suffix}"
            if value.endswith(f"_{suffix}"):
                return value
            return f"{value}_{suffix}"

        @classmethod
        def spatial_dist(cls, value: str | None = None) -> str:
            return cls._spatial_key(value, "distances")

        @classmethod
        def spatial_conn(cls, value: str | None = None) -> str:
            return cls._spatial_key(value, "connectivities")

    class uns:
        @classmethod
        def spatial_neighs(cls, value: str | None = None) -> str:
            return f"{Key.obsm.spatial}_neighbors" if value is None else f"{value}_neighbors"

        @classmethod
        def ligrec(cls, cluster: str, value: str | None = None) -> str:
            return f"{cluster}_ligrec" if value is None else value

        @classmethod
        def nhood_enrichment(cls, cluster: str) -> str:
            return f"{cluster}_nhood_enrichment"

        @classmethod
        def co_occurrence(cls, cluster: str) -> str:
            return f"{cluster}_co_occurrence"

        @classmethod
        def ripley(cls, cluster: str, mode) -> str:
            return f"{cluster}_ripley_{mode}"

        @classmethod
        def centrality_scores(cls, cluster: str) -> str:
            return f"{cluster}_centrality_scores"

        @classmethod
        def interaction_matrix(cls, cluster: str) -> str:
            return f"{cluster}_interactions"
