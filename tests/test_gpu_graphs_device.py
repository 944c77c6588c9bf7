"""Spatial graphs built from coordinates in GPU memory (``sqb_graph_build_device``): for every golden case and builder option
the device result (torch ``sparse_csr`` CUDA tensors) equals the host builders' result after ``sort_indices()`` -- same
indptr / indices, same dtype, values bit for bit -- and the reference golden; torch f64 / f32 tensors, strided views and a
``__cuda_array_interface__`` duck type that must never be read on the host; ``library_key``; the 1M-spot lattice; a
device-built graph feeding the statistics; producer streams; errors leave the context usable."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200.gr import GridBuilder, KNNBuilder, RadiusBuilder  # noqa: E402
from tests.golden.make_golden_graphs import cases  # noqa: E402
from tests.test_gpu_graphs import GOLD, _check  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu
BUILDERS = {"KNNBuilder": KNNBuilder, "GridBuilder": GridBuilder, "RadiusBuilder": RadiusBuilder}


class CuCoords:
    """cupy-like device array behind a version-3 interface; converting it on the host fails the test."""

    def __init__(self, t, stream=None):
        self.t, self.stream = t, stream

    @property
    def shape(self):
        return tuple(self.t.shape)

    @property
    def __cuda_array_interface__(self):
        d = dict(self.t.__cuda_array_interface__)
        d.update(version=3, stream=self.stream)
        return d

    def __array__(self, *a, **k):
        raise AssertionError("device coordinates were read on the host")


def _scipy(t) -> sp.csr_matrix:
    assert t.layout == torch.sparse_csr and t.is_cuda
    assert t.crow_indices().dtype == torch.int32 and t.col_indices().dtype == torch.int32
    c = t.cpu()
    return sp.csr_matrix((c.values().numpy(), c.col_indices().numpy(), c.crow_indices().numpy()), shape=tuple(t.shape))


def _same(dev, host):
    for tag, t, h in (("adj", dev[0], host[0]), ("dst", dev[1], host[1])):
        m, h = _scipy(t), h.tocsr()
        h.sort_indices()
        np.testing.assert_array_equal(m.indptr, h.indptr, err_msg=f"{tag} indptr")
        np.testing.assert_array_equal(m.indices, h.indices, err_msg=f"{tag} indices")
        assert m.data.dtype == h.data.dtype, (tag, m.data.dtype, h.data.dtype)
        assert m.data.tobytes() == h.data.tobytes(), f"{tag} data differ"


def _variants(co):
    """(name, device coordinates, host coordinates they hold)"""
    t = torch.tensor(co, device="cuda")
    strided = torch.zeros((co.shape[0], 2, 3), dtype=torch.float64, device="cuda")[:, :, 1]
    strided.copy_(t)
    co32 = co.astype(np.float32).astype(np.float64)
    return [("f64", t, co), ("strided", strided, co), ("cai", CuCoords(t), co), ("f32", torch.tensor(co32, dtype=torch.float32, device="cuda"), co32)]


@pytest.mark.parametrize("name", list(cases()))
def test_golden_cases_device_equal_host_and_reference(name):
    co, cls, kw = cases()[name]
    for tag, dev_co, host_co in _variants(co):
        dev = BUILDERS[cls](**kw).build(dev_co)
        _same(dev, BUILDERS[cls](**kw).build(host_co.copy()))
        if tag != "f32":
            _check(name, _scipy(dev[0]), _scipy(dev[1]), exact_adj=kw.get("transform") is None)


OPTIONS = {
    "knn_pct_nodiag": (KNNBuilder, dict(n_neighs=6, percentile=80.0)),
    "knn_pct_diag": (KNNBuilder, dict(n_neighs=6, percentile=80.0, set_diag=True)),
    "knn_pct_q100": (KNNBuilder, dict(n_neighs=3, percentile=100.0)),
    "knn_diag_spectral": (KNNBuilder, dict(n_neighs=9, set_diag=True, transform="spectral")),
    "knn_pct_cosine": (KNNBuilder, dict(n_neighs=6, percentile=90.0, transform="cosine")),
    "knn_diag_cosine": (KNNBuilder, dict(n_neighs=5, set_diag=True, transform="cosine")),
    "radius_pct_diag": (RadiusBuilder, dict(radius=30.0, percentile=37.5, set_diag=True)),
    "radius_interval_diag": (RadiusBuilder, dict(radius=(5.0, 20.0), set_diag=True)),
    "radius_interval_pct_cosine": (RadiusBuilder, dict(radius=(5.0, 30.0), percentile=60.0, transform="cosine")),
    "grid_rings3": (GridBuilder, dict(n_neighs=6, n_rings=3)),
    "grid_rings3_diag": (GridBuilder, dict(n_neighs=6, n_rings=3, set_diag=True)),
    "grid_rings4_spectral": (GridBuilder, dict(n_neighs=6, n_rings=4, transform="spectral")),
    "grid_rings4_diag_cosine": (GridBuilder, dict(n_neighs=4, n_rings=4, set_diag=True, transform="cosine")),
}


@pytest.mark.parametrize("name", list(OPTIONS))
@pytest.mark.parametrize("coords", ["uniform", "clustered", "hex"])
def test_options_device_equal_host(name, coords):
    rng = np.random.default_rng(3)
    co = {"uniform": rng.random((2000, 2)) * 700.0,
          "clustered": (rng.random((8, 2)) * 500.0)[rng.integers(0, 8, 1500)] + rng.normal(0.0, 15.0, (1500, 2)),
          "hex": synth.hex_coords(30, 37, scale=10.0)}[coords]
    cls, kw = OPTIONS[name]
    _same(cls(**kw).build(torch.tensor(co, device="cuda")), cls(**kw).build(co.copy()))


def _lib_adata(co, codes, n_cat):
    obs = pd.DataFrame({"lib": pd.Categorical.from_codes(codes, categories=[f"l{i}" for i in range(n_cat)])}, index=[str(i) for i in range(len(codes))])
    return sq.AnnDataLite(obs=obs, obsm={"spatial": co}, shape=(len(codes), 0))


def test_library_key_golden_and_four_libraries():
    co, codes = GOLD["lib_coords"], GOLD["lib_codes"]
    res = sq.gr.spatial_neighbors_knn(_lib_adata(torch.tensor(co, device="cuda"), codes, 2), n_neighs=5, library_key="lib", copy=True)
    _check("lib", _scipy(res.connectivities), _scipy(res.distances))
    rng = np.random.default_rng(4)
    co4 = rng.random((3000, 2)) * 400.0
    codes4 = rng.integers(0, 4, 3000)
    for fn, kw in ((sq.gr.spatial_neighbors_knn, dict(n_neighs=6, percentile=90.0, set_diag=True)),
                   (sq.gr.spatial_neighbors_knn, dict(n_neighs=4, transform="cosine")),
                   (sq.gr.spatial_neighbors_grid, dict(n_neighs=6, n_rings=3, transform="spectral")),
                   (sq.gr.spatial_neighbors_radius, dict(radius=(2.0, 15.0), percentile=75.0))):
        dev = fn(_lib_adata(CuCoords(torch.tensor(co4, device="cuda")), codes4, 4), library_key="lib", copy=True, **kw)
        host = fn(_lib_adata(co4, codes4, 4), library_key="lib", copy=True, **kw)
        _same(dev, host)


def test_spatial_neighbors_writes_device_obsp():
    co = synth.hex_coords(20, 25)
    ad = synth.make_adata(torch.tensor(co, device="cuda"), None, None)
    sq.gr.spatial_neighbors_grid(ad, n_neighs=6)
    g = ad.obsp["spatial_connectivities"]
    assert g.layout == torch.sparse_csr and g.device == torch.device("cuda", 0) and g.values().dtype == torch.float32
    assert (_scipy(g) != synth.hex_graph(20, 25)).nnz == 0
    assert ad.uns["spatial_neighbors"]["params"]["coord_type"] == "grid"


def test_large_lattices_device_equal_host():
    co = synth.hex_coords(1000, 1000)
    t = torch.tensor(co, device="cuda")
    for b in (GridBuilder(6), KNNBuilder(6, set_diag=True, percentile=99.0)):
        _same(b.build(t), b.build(co))
    co2 = synth.hex_coords(450, 450)
    _same(GridBuilder(6, n_rings=3).build(torch.tensor(co2, device="cuda")), GridBuilder(6, n_rings=3).build(co2))


def _eq(a, b):
    if isinstance(a, pd.DataFrame):
        pd.testing.assert_frame_equal(a, b, check_exact=True)
    elif isinstance(a, tuple):
        for x, y in zip(a, b, strict=True):
            _eq(x, y)
    else:
        np.testing.assert_array_equal(np.asarray(a), np.asarray(b))


def test_pipeline_device_coordinates_to_statistics():
    rows, cols = 40, 45
    co = synth.hex_coords(rows, cols)
    n = co.shape[0]
    rng = np.random.default_rng(9)
    labels = pd.Series(pd.Categorical.from_codes(rng.integers(0, 5, n), categories=[f"c{i}" for i in range(5)]))
    x = rng.poisson(1.0, (n, 6)).astype(np.float64)
    out = {}
    for tag, coords in (("host", co), ("device", torch.tensor(co, device="cuda"))):
        ad = synth.make_adata(coords, None, labels, X=x)
        sq.gr.spatial_neighbors_grid(ad, n_neighs=6)
        assert (tag == "device") == isinstance(ad.obsp["spatial_connectivities"], torch.Tensor)
        out[tag] = (tuple(sq.gr.nhood_enrichment(ad, "cluster", n_perms=50, seed=3, copy=True)),
                    sq.gr.interaction_matrix(ad, "cluster", copy=True),
                    sq.gr.spatial_autocorr(ad, mode="moran", copy=True),
                    sq.gr.sepal(ad, max_neighs=6, n_iter=2000, copy=True),
                    tuple(sq.gr.co_occurrence(ad, "cluster", interval=8, copy=True)))
    _eq(out["device"], out["host"])


def test_producer_stream_is_honoured():
    co = np.random.default_rng(1).random((200_000, 2)) * 5000.0
    src = torch.tensor(co, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        t = torch.zeros_like(src)
        torch.cuda._sleep(50_000_000)  # the copy below lands long after the call has been issued
        t.copy_(src)
    res = KNNBuilder(6).build(CuCoords(t, stream=s.cuda_stream))
    _same(res, KNNBuilder(6).build(co))
    torch.cuda.synchronize()


def test_errors_raise_and_context_stays_usable():
    co = np.random.default_rng(2).random((50, 2)) * 10.0
    bad = co.copy()
    bad[17, 1] = np.nan
    bad[30, 0] = np.inf
    with pytest.raises(ValueError, match="observation 17 are not finite"):
        KNNBuilder(4).build(torch.tensor(bad, device="cuda"))
    with pytest.raises(ValueError, match="n_neighbors"):
        KNNBuilder(50).build(torch.tensor(co, device="cuda"))
    with pytest.raises(NotImplementedError, match=r"outside \[1, 64\]"):
        KNNBuilder(65).build(torch.tensor(np.random.default_rng(0).random((100, 2)), device="cuda"))
    with pytest.raises(ValueError, match="shape"):
        KNNBuilder(4).build(torch.zeros((50, 3), dtype=torch.float64, device="cuda"))
    with pytest.raises(TypeError, match="dtype"):
        KNNBuilder(4).build(torch.zeros((50, 2), dtype=torch.int32, device="cuda"))
    ad = synth.make_adata(torch.tensor(co, device="cuda"), None, None)
    with pytest.raises(ValueError, match="does not match the device"):
        sq.gr.spatial_neighbors_knn(ad, n_neighs=4, device=torch.cuda.device_count())
    with pytest.raises(NotImplementedError):
        sq.gr.spatial_neighbors_grid(ad, delaunay=True)
    sq.gr.spatial_neighbors_knn(ad, n_neighs=4)
    _same((ad.obsp["spatial_connectivities"], ad.obsp["spatial_distances"]), KNNBuilder(4).build(co))
