"""Every device buffer the library takes from the stream-ordered allocator is returned by the end of the call that took it:
after repeated successful calls of every family, and after every input error the library detects on the device once its
buffers exist, the bytes in use in the device's default memory pool are back where they were.

The count comes from the driver: ``cuMemPoolGetAttribute(CU_MEMPOOL_ATTR_USED_MEM_CURRENT)`` of ``cuDeviceGetDefaultMemPool``.
The pool is a per-device driver object, so the count does not depend on how the library resolves cudart.  It covers this
process's stream-ordered allocations only: work of other processes on a shared GPU does not move it, and torch's caching
allocator does not use that pool."""

from __future__ import annotations

import ctypes
import gc

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200 import AnnDataLite  # noqa: E402
from squidpy_b200._lib import check, load  # noqa: E402
from squidpy_b200.gr import AutocorrPlan, GridBuilder, KNNBuilder, NhoodPlan, RadiusBuilder  # noqa: E402
from tests.test_gpu_autocorr_device_input import CuSparse  # noqa: E402
from tests.test_gpu_autocorr_device_input import _adata as _ac_adata  # noqa: E402
from tests.test_gpu_autocorr_device_input import _corrupt as _ac_corrupt  # noqa: E402
from tests.test_gpu_autocorr_device_input import _w  # noqa: E402
from tests.test_gpu_autocorr_device_input import _x as _ac_x  # noqa: E402
from tests.test_gpu_ligrec_sepal_device_input import GENES, _dev, _ligrec_dev, _sepal_adata, _sepal_x  # noqa: E402
from tests.test_gpu_ligrec_sepal_device_input import _x as _lr_x  # noqa: E402
from tests.test_gpu_nhood_device_graph import _adata as _nh_adata  # noqa: E402
from tests.test_gpu_nhood_device_graph import _corrupt as _nh_corrupt  # noqa: E402
from tests.test_gpu_nhood_device_graph import _graph  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu
CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7
REPEATS = 10


def _pool_used() -> int:
    cu = ctypes.CDLL("libcuda.so.1")
    dev, pool, used = ctypes.c_int(), ctypes.c_void_p(), ctypes.c_uint64()
    assert cu.cuInit(0) == 0
    assert cu.cuDeviceGet(ctypes.byref(dev), sq.default_context().device) == 0
    assert cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, ctypes.byref(used)) == 0
    return used.value


def _settled_pool_used() -> int:
    gc.collect()  # handles still referenced by dropped results are closed here
    torch.cuda.synchronize()  # stream-ordered frees take effect in stream order
    return _pool_used()


def _raises(exc, match, call):
    def run():
        with pytest.raises(exc, match=match):
            call()

    return run


# ---- successful calls --------------------------------------------------------------------------------------------------
def _nhood(graph, **kw):
    g = _graph("knn")
    return lambda: sq.gr.nhood_enrichment(_nh_adata(graph(g), g.shape[0], 5), "cl", n_perms=20, seed=1, copy=True, **kw)


def _interaction(graph, **kw):
    g = _graph("messy")
    return lambda: sq.gr.interaction_matrix(_nh_adata(graph(g), g.shape[0], 6, nan=True), "cl", copy=True, **kw)


def _ligrec(device):
    x = _lr_x(n=300, seed=2)
    return lambda: _ligrec_dev(_dev(x, "csr") if device else x, 300)


def _sepal(device):
    x = _sepal_x(14 * 15)
    return lambda: sq.gr.sepal(_sepal_adata(_dev(x, "csr") if device else sp.csr_matrix(x), x.shape[1]), max_neighs=6, n_iter=300, copy=True)


def _autocorr(device, **kw):
    w = _w()
    x = _ac_x(w.shape[0], g=12)
    return lambda: sq.gr.spatial_autocorr(_ac_adata(CuSparse.of(x) if device else x, w, 12), mode="moran", copy=True, **kw)


def _autocorr_dense_device():
    w = _w()
    x = _ac_x(w.shape[0], g=12).toarray()
    return lambda: sq.gr.spatial_autocorr(_ac_adata(torch.as_tensor(x).cuda(), w, 12), mode="geary", copy=True)


def _builder(cls, device, **kw):
    co = np.random.default_rng(3).random((1500, 2)) * 500.0
    return lambda: cls(**kw).build(torch.tensor(co, device="cuda") if device else co.copy())


def _knn_libraries():
    rng = np.random.default_rng(4)
    co, codes = rng.random((2000, 2)) * 400.0, rng.integers(0, 4, 2000)
    obs = pd.DataFrame({"lib": pd.Categorical.from_codes(codes, categories=[f"l{i}" for i in range(4)])}, index=[str(i) for i in range(2000)])
    return lambda: sq.gr.spatial_neighbors_knn(AnnDataLite(obs=obs, obsm={"spatial": torch.tensor(co, device="cuda")}, shape=(2000, 0)),
                                               n_neighs=5, library_key="lib", copy=True)


# ---- input errors detected on the device -------------------------------------------------------------------------------
def _nhood_host_invalid_csr():
    return _raises(ValueError, "invalid CSR", lambda: NhoodPlan(np.array([0, 1, 2, 3]), np.array([1, 7, 0]), 2))


def _first_indptr(g):
    ip = g.indptr.copy()
    ip[0] = 1
    return ip


def _big_index(g):
    ix = g.indices.copy()
    ix[17] = g.shape[0]
    return ix


def _nhood_device_error(array, match):
    g = _graph("knn")
    _, dev = _nh_corrupt(g, **array(g))
    return _raises(ValueError, match, lambda: sq.gr.nhood_enrichment(_nh_adata(dev, g.shape[0], 3), "cl", n_perms=8, seed=1, copy=True))


def _interaction_device_error(array, match):
    g = _graph("knn")
    _, dev = _nh_corrupt(g, **array(g))
    return _raises(ValueError, match, lambda: sq.gr.interaction_matrix(_nh_adata(dev, g.shape[0], 3), "cl", copy=True))


def _interaction_code_out_of_range():
    """Codes come from a categorical in sq.gr.interaction_matrix, so a code >= n_cls only reaches the library directly."""
    g = synth.hex_graph(20, 20)
    n = g.shape[0]
    ip, ix = (torch.as_tensor(a.astype(np.int32)).cuda() for a in (g.indptr, g.indices))
    codes = np.zeros(n, np.int32)
    codes[7] = 3
    out = np.zeros((3, 3), np.int64)

    def call():
        torch.cuda.synchronize()  # the tensors are complete: no producer stream is named
        ctx = sq.default_context()
        with ctx.lock:
            check(load().sqb_interaction_matrix_device(ctx.handle, n, g.nnz, ip.data_ptr(), 32, ix.data_ptr(), 32, None, 0, codes.ctypes.data,
                                                       3, None, out.ctypes.data, 0))

    return _raises(ValueError, "a code is >= n_cls", call)


def _ligrec_error(kind):
    """The invalid expression matrices of test_gpu_ligrec_sepal_device_input.test_errors_leave_the_context_usable."""
    x = _lr_x(n=300, seed=13)
    m = sp.csr_matrix(x)
    col = GENES.index("Il2")
    if kind == "duplicate_cell":  # row 0 stores Il2 twice
        x0 = x.copy()
        x0[0, col] = 2.0
        m0 = sp.csr_matrix(x0)
        a = m0.indptr[1]
        ip = m0.indptr.astype(np.int32).copy()
        ip[1:] += 1
        bad = CuSparse("csr", ip, np.insert(m0.indices, a, col).astype(np.int32), np.insert(m0.data, a, np.float32(1.0)), m0.shape)
        return _raises(ValueError, "same gathered cell", lambda: _ligrec_dev(bad, 300))
    if kind == "index_out_of_range":
        ix = m.indices.astype(np.int32).copy()
        ix[m.indices == col] = len(GENES) + 5
        bad = CuSparse("csr", m.indptr.astype(np.int32), ix, m.data, m.shape)
        return _raises(ValueError, "out of range", lambda: _ligrec_dev(bad, 300))
    ip = m.indptr.astype(np.int64).copy()
    ip[5], ip[6] = ip[6] + 1, ip[5]
    bad = CuSparse("csr", ip, m.indices.astype(np.int32), m.data, m.shape)
    return _raises(ValueError, "indptr", lambda: _ligrec_dev(bad, 300))


def _sepal_indptr():
    ms = sp.csr_matrix(_sepal_x(14 * 15))
    ip = ms.indptr.astype(np.int64).copy()
    ip[5], ip[6] = ip[6] + 1, ip[5]
    x = CuSparse("csr", ip, ms.indices, ms.data, ms.shape)
    return _raises(ValueError, "indptr", lambda: sq.gr.sepal(_sepal_adata(x, 9), max_neighs=6, n_iter=10, copy=True))


def _autocorr_error(where, kind):
    """The invalid feature matrices of test_gpu_autocorr_device_input.test_invalid_input_raises_like_the_host_and_context_survives,
    on the host (checked on the device while the matrix is re-laid out) and in device memory.  where="host_by_feature": the
    host CSR of features x observations, loaded as such (layout 0 of sqb_autocorr_load_csr)."""
    w = _w()
    x = _ac_x(w.shape[0], g=10, density=0.3)
    if where == "host_by_feature":
        x = x.T.tocsr()
    r = int(np.flatnonzero(np.diff(x.indptr) >= 2)[0])
    a = x.indptr[r]
    if kind == "duplicate":
        ix = x.indices.copy()
        ix[a + 1] = ix[a]
        arrays, match = {"indices": ix}, "stored twice"
    elif kind == "index_out_of_range":
        ix = x.indices.copy()
        ix[a] = x.shape[1]
        arrays, match = {"indices": ix}, "out of range"
    else:
        ip = x.indptr.copy()
        ip[r + 1] = ip[r] - 1 if ip[r] > 0 else ip[r + 2] + 1
        arrays, match = {"indptr": ip}, "indptr"
    host, dev = _ac_corrupt(x, **arrays)
    if where == "host_by_feature":

        def load():
            plan = AutocorrPlan(w)
            try:
                plan.load(host, obs_major=False)
            finally:
                plan.close()

        return _raises(ValueError, match, load)
    m = host if where == "host" else dev
    return _raises(ValueError, match, lambda: sq.gr.spatial_autocorr(_ac_adata(m, w, 10), copy=True))


# name -> factory of the call (built inside the test: nothing touches the GPU at import)
CASES = {
    "nhood_exact_host_graph": lambda: _nhood(lambda g: g),
    "nhood_exact_device_graph": lambda: _nhood(CuSparse.of),
    "nhood_philox_host_graph": lambda: _nhood(lambda g: g, rng="philox"),
    "nhood_philox_device_graph": lambda: _nhood(CuSparse.of, rng="philox"),
    "ligrec_host_x": lambda: _ligrec(False),
    "ligrec_device_x": lambda: _ligrec(True),
    "sepal_host_x": lambda: _sepal(False),
    "sepal_device_x": lambda: _sepal(True),
    "autocorr_host_x": lambda: _autocorr(False),
    "autocorr_host_x_perms": lambda: _autocorr(False, n_perms=5, seed=2),
    "autocorr_device_x": lambda: _autocorr(True),
    "autocorr_device_dense_x": _autocorr_dense_device,
    "interaction_host_graph": lambda: _interaction(lambda g: g),
    "interaction_host_graph_weights": lambda: _interaction(lambda g: g, weights=True),
    "interaction_device_graph": lambda: _interaction(CuSparse.of),
    "interaction_device_graph_weights": lambda: _interaction(CuSparse.of, weights=True),
    "knn_host_coords": lambda: _builder(KNNBuilder, False, n_neighs=6),
    "knn_device_coords": lambda: _builder(KNNBuilder, True, n_neighs=6),
    "knn_device_coords_percentile_cosine": lambda: _builder(KNNBuilder, True, n_neighs=6, percentile=90.0, transform="cosine"),
    "knn_device_coords_libraries": _knn_libraries,
    "radius_host_coords": lambda: _builder(RadiusBuilder, False, radius=30.0),
    "radius_device_coords": lambda: _builder(RadiusBuilder, True, radius=30.0),
    "radius_device_coords_interval_spectral": lambda: _builder(RadiusBuilder, True, radius=(5.0, 30.0), set_diag=True, transform="spectral"),
    "grid_host_coords": lambda: _builder(GridBuilder, False, n_neighs=6),
    "grid_device_coords": lambda: _builder(GridBuilder, True, n_neighs=6),
    "grid_device_coords_rings": lambda: _builder(GridBuilder, True, n_neighs=6, n_rings=3, set_diag=True),
    # input errors detected on the device after the call has allocated
    "nhood_host_invalid_csr": _nhood_host_invalid_csr,
    "nhood_device_indptr": lambda: _nhood_device_error(lambda g: {"indptr": _first_indptr(g)}, "indptr"),
    "nhood_device_index_out_of_range": lambda: _nhood_device_error(lambda g: {"indices": _big_index(g)}, "invalid CSR"),
    "interaction_device_indptr": lambda: _interaction_device_error(lambda g: {"indptr": _first_indptr(g)}, "indptr"),
    "interaction_device_index_out_of_range": lambda: _interaction_device_error(lambda g: {"indices": _big_index(g)}, "out of range"),
    "interaction_device_code_out_of_range": _interaction_code_out_of_range,
    "ligrec_duplicate_cell": lambda: _ligrec_error("duplicate_cell"),
    "ligrec_index_out_of_range": lambda: _ligrec_error("index_out_of_range"),
    "ligrec_indptr": lambda: _ligrec_error("indptr"),
    "sepal_device_indptr": _sepal_indptr,
    **{f"autocorr_{where}_{kind}": (lambda where=where, kind=kind: _autocorr_error(where, kind))
       for where in ("host", "host_by_feature", "device") for kind in ("duplicate", "index_out_of_range", "indptr")},
}


@pytest.mark.parametrize("case", list(CASES))
def test_pool_bytes_return_to_baseline(case):
    call = CASES[case]()
    call()  # warm-up: module loading, lazily built tables, the context's first use
    base = _settled_pool_used()
    for _ in range(REPEATS):
        call()
    assert _settled_pool_used() == base
