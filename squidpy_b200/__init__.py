"""squidpy_b200 — H100-native (sm_90a CUDA) implementation of squidpy's spatial-statistics hot path:
``gr.nhood_enrichment``, ``gr.spatial_autocorr`` (Moran's I / Geary's C), ``gr.co_occurrence``, ``gr.ripley``, and
``tl.var_by_distance``.

Drop-in for the same-named ``squidpy.gr`` / ``squidpy.tl`` functions (same signatures, same AnnData keys); the numeric hot loops run
in ``libsquidpy_b200.so`` through a ctypes C ABI (``include/squidpy_b200.h``).  There is no CPU fallback.
"""

from . import gr, tl
from ._adata import AnnDataLite
from ._lib import Context, SquidpyB200Error, default_context, device_count, set_default_context

__version__ = "0.1.0"
__all__ = ["gr", "tl", "AnnDataLite", "Context", "SquidpyB200Error", "default_context", "set_default_context", "device_count", "__version__"]
