"""``spatial_neighbors`` and custom builders on the GPU: every resolution branch equals the matching ``spatial_neighbors_*``
call on host and device coordinates, the reference's known answers hold, and a custom ``GraphBuilderCSR`` on device
coordinates (never read on the host) builds per library on the device and combines there, equal to the host result."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

import squidpy_b200 as sq  # noqa: E402
from squidpy_b200._constants import Transform  # noqa: E402
from squidpy_b200.gr import neighbors as nb  # noqa: E402
from tests.test_gpu_graph_postprocess import to_host  # noqa: E402
from tests.test_gpu_graphs_device import CuCoords  # noqa: E402
from tests.test_neighbors_api_host import GOLD, assert_same_csr  # noqa: E402

pytestmark = pytest.mark.gpu

RNG = np.random.default_rng(11)
CO = RNG.uniform(0, 200, (600, 2))
CODES = RNG.integers(0, 3, 600)

BRANCHES = [  # (spatial_neighbors kwargs, "spatial" in uns, the matching call)
    (dict(), False, (sq.gr.spatial_neighbors_knn, dict())),
    (dict(n_neighs=8, percentile=70.0, transform="cosine"), False, (sq.gr.spatial_neighbors_knn, dict(n_neighs=8, percentile=70.0, transform="cosine"))),
    (dict(radius=12.0, set_diag=True), False, (sq.gr.spatial_neighbors_radius, dict(radius=12.0, set_diag=True))),
    (dict(coord_type="generic", radius=(3.0, 12.0), transform="spectral"), True,
     (sq.gr.spatial_neighbors_radius, dict(radius=(3.0, 12.0), transform="spectral"))),
    (dict(delaunay=True, radius=9.0), False, (sq.gr.spatial_neighbors_delaunay, dict())),
    (dict(delaunay=True, radius=(2.0, 15.0), percentile=80.0), False, (sq.gr.spatial_neighbors_delaunay, dict(radius=(2.0, 15.0), percentile=80.0))),
    (dict(), True, (sq.gr.spatial_neighbors_grid, dict())),
    (dict(coord_type="grid", n_neighs=4, n_rings=3, transform="cosine"), False,
     (sq.gr.spatial_neighbors_grid, dict(n_neighs=4, n_rings=3, transform="cosine"))),
]


def _adata(co, uns=False, codes=None):
    obs = None if codes is None else pd.DataFrame({"lib": pd.Categorical.from_codes(codes, ["a", "b", "c"])})
    return sq.AnnDataLite(obs=obs, obsm={"spatial": co}, uns={"spatial": {}} if uns else None, shape=(co.shape[0], 0))


def _as_host(m):
    return to_host(m) if isinstance(m, torch.Tensor) else sp.csr_matrix(m)


@pytest.mark.parametrize("i", range(len(BRANCHES)))
@pytest.mark.parametrize("where", ["host", "device"])
def test_spatial_neighbors_equals_the_matching_call(i, where):
    kw, uns, (fn, fkw) = BRANCHES[i]
    co = CO if where == "host" else CuCoords(torch.tensor(CO, device="cuda"))
    for lib in (None, "lib"):
        with pytest.warns(FutureWarning):
            got = sq.gr.spatial_neighbors(_adata(co, uns, CODES), library_key=lib, copy=True, **kw)
        want = fn(_adata(co, uns, CODES), library_key=lib, copy=True, **fkw)
        assert_same_csr(_as_host(got.connectivities), _as_host(want.connectivities))
        assert_same_csr(_as_host(got.distances), _as_host(want.distances))
    adata = _adata(co, uns)
    with pytest.warns(FutureWarning):
        sq.gr.spatial_neighbors(adata, **kw)
    ref = _adata(co, uns)
    fn(ref, **fkw)
    assert adata.uns["spatial_neighbors"]["params"] == ref.uns["spatial_neighbors"]["params"]


@pytest.mark.parametrize("where", ["host", "device"])
def test_known_answers(where):
    vis = GOLD["known/visium_coords"].astype(np.float64)
    grid = GOLD["known/squaregrid_coords"].astype(np.float64)
    put = (lambda a: a) if where == "host" else (lambda a: torch.tensor(a, device="cuda"))
    for n_rings, conn, dist in GOLD["known/visium_rings_conn_dist"]:
        adata = _adata(put(vis), uns=True)
        with pytest.warns(FutureWarning):
            sq.gr.spatial_neighbors(adata, n_rings=int(n_rings))
        a, d = _as_host(adata.obsp["spatial_connectivities"]), _as_host(adata.obsp["spatial_distances"])
        assert a[0].sum() == conn
        if n_rings > 1:
            assert d[0].sum() == dist
    for n_rings, degree in GOLD["known/squaregrid_rings_degree"]:
        adata = _adata(put(grid))
        with pytest.warns(FutureWarning):
            sq.gr.spatial_neighbors(adata, n_neighs=4, n_rings=int(n_rings), coord_type="grid")
        assert np.diff(_as_host(adata.obsp["spatial_connectivities"]).indptr).max() == degree


class DeviceKNN(nb.GraphBuilderCSR):
    """A caller's builder whose graph is the built-in kNN graph, post-processed by the public classes."""

    def __init__(self, percentile=None, transform=None):
        steps = [] if percentile is None else [nb.PercentilePostprocessor(percentile)]
        super().__init__(transform=transform, percentile=percentile, postprocessors=[*steps, nb.TransformPostprocessor(Transform.NONE if transform is None else Transform(transform))])
        self.seen = []

    def build_graph(self, coords):
        self.seen.append(type(coords))
        return nb.KNNBuilder(n_neighs=5).build(coords)

    def uns_params(self):
        return {"coord_type": "generic", "transform": self.transform.v}


@pytest.mark.parametrize("lib", [None, "lib"])
def test_custom_builder_on_device_coordinates(lib):
    dev_builder, host_builder = DeviceKNN(percentile=70.0, transform="cosine"), DeviceKNN(percentile=70.0, transform="cosine")
    got = sq.gr.spatial_neighbors_from_builder(_adata(CuCoords(torch.tensor(CO, device="cuda")), codes=CODES), dev_builder, library_key=lib, copy=True)
    want = sq.gr.spatial_neighbors_from_builder(_adata(CO, codes=CODES), host_builder, library_key=lib, copy=True)
    assert got.connectivities.is_cuda and got.distances.is_cuda
    assert len(dev_builder.seen) == (1 if lib is None else 3)
    assert_same_csr(to_host(got.connectivities), sp.csr_matrix(want.connectivities))
    assert_same_csr(to_host(got.distances), sp.csr_matrix(want.distances))


def test_custom_builder_mixing_host_and_device_matrices_is_refused():
    class Mixed(nb.GraphBuilderCSR):
        def build_graph(self, coords):
            adj, dst = nb.KNNBuilder(n_neighs=3).build(coords)
            return adj, sp.csr_matrix(to_host(dst))

        def uns_params(self):
            return {}

    with pytest.raises(TypeError, match="one on the host"):
        sq.gr.spatial_neighbors_from_builder(_adata(torch.tensor(CO, device="cuda")), Mixed())
