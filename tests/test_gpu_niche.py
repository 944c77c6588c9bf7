"""calculate_niche on the GPU: the device embeddings against the numpy restatement (bit for bit) and the public functions
against the reference's golden, through the recording scanpy stand-in."""

from __future__ import annotations

import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

from squidpy_b200.gr import _niche
from tests import niche_ref
from tests import niche_scanpy_standin as standin
from tests.golden.make_golden_niche import build_call, cases, graphs, make_adata, run
from tools import synth

pytestmark = pytest.mark.gpu

GOLD = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "niche.npz"), allow_pickle=False))
CASES = cases()
GRAPHS = graphs()


def _is_cellcharter(case):
    return case[1] == "cellcharter" or case[3].get("flavor") == "cellcharter"


@pytest.mark.parametrize("i", range(len(CASES)), ids=[c[0] for c in CASES])
def test_public_functions_match_golden(i):
    from sklearn.mixture import GaussianMixture

    case = CASES[i]
    standin.install()
    adata, kw = build_call(case, GRAPHS)
    before = set(adata.obs.columns)
    res, calls = run(_niche, case[1], adata, kw)
    assert len(calls) == int(GOLD[f"c{i}_ncalls"])
    for j, (name, X, info) in enumerate(calls):
        assert name == str(GOLD[f"c{i}_k{j}_name"])
        assert info == json.loads(str(GOLD[f"c{i}_k{j}_info"]))
        G = GOLD[f"c{i}_k{j}_X"]
        if _is_cellcharter(case) and name == "pca":
            m = adata.n_vars
            np.testing.assert_array_equal(X[:, : 2 * m], G[:, : 2 * m])  # X and hop 1: bit for bit
            np.testing.assert_allclose(X[:, 2 * m:], G[:, 2 * m:], rtol=1e-12, atol=1e-300)
        elif "weighted" in case[0] and case[1] == "neighborhood":
            np.testing.assert_allclose(X, G, rtol=1e-5)
        else:
            np.testing.assert_array_equal(X, G)
    cols = sorted(set(res.obs.columns) - before)
    assert cols == list(GOLD[f"c{i}_cols"])
    for j, col in enumerate(cols):
        got = res.obs[col].astype(str).to_numpy()
        if _is_cellcharter(case) and "use_rep" not in case[3] and "library_key" not in case[3] and col == "cellcharter_niche":
            # the GMM runs on this host's BLAS: pin the labels to the same GMM on the golden's PCA input
            Y = standin.pca_of(GOLD[f"c{i}_k0_X"])
            gmm = GaussianMixture(n_components=kw["n_components"], random_state=kw.get("random_state", 42), init_params="random_from_data")
            expect = gmm.fit(Y).predict(Y).astype(str)
            np.testing.assert_array_equal(got, expect)
        else:
            np.testing.assert_array_equal(got, GOLD[f"c{i}_col{j}"])


def _codes(adata):
    col = adata.obs["cell_type"]
    return col.cat.codes.to_numpy().astype(np.int32), len(col.cat.categories)


@pytest.mark.parametrize("g", sorted(GRAPHS))
@pytest.mark.parametrize("distance,weights,abs_nhood", [(1, None, False), (2, None, True), (3, [1.0, 0.5], False), (4, [2, 1, 0.5], True)])
def test_profile_kernel_matches_restatement(g, distance, weights, abs_nhood):
    A = GRAPHS[g]
    adata = make_adata(A)
    codes, C = _codes(adata)
    got = _niche.niche_profile(A, codes, C, distance, weights, abs_nhood)
    np.testing.assert_array_equal(got, niche_ref.profile(A, codes, C, distance, weights, abs_nhood))


@pytest.mark.parametrize("g", sorted(GRAPHS))
@pytest.mark.parametrize("xkind", ["sparse32", "dense32", "dense64", "sparse64"])
def test_utag_kernel_matches_restatement(g, xkind):
    A = GRAPHS[g]
    adata = make_adata(A, sparse_x=xkind.startswith("sparse"), x_dtype=np.float32 if xkind.endswith("32") else np.float64)
    got, _ = _niche.niche_aggregate(A, adata.X, "utag")
    expect = niche_ref.utag(A, adata.X)
    assert got.dtype == expect.dtype
    np.testing.assert_array_equal(got, expect)


@pytest.mark.parametrize("g", sorted(GRAPHS))
@pytest.mark.parametrize("aggregation", ["mean", "variance"])
@pytest.mark.parametrize("distance", [1, 2, 4])
def test_cellcharter_kernel_matches_restatement(g, aggregation, distance):
    A = GRAPHS[g]
    adata = make_adata(A)
    got, nnz = _niche.niche_aggregate(A, adata.X, aggregation, distance)
    expect, expect_nnz = niche_ref.cellcharter(A, adata.X, distance, aggregation)
    assert got.dtype == expect.dtype and list(nnz) == expect_nnz
    np.testing.assert_array_equal(got, expect)


def test_hop_sets_on_long_rows():
    """Rows whose hop product exceeds the shared-memory table use the global-memory one; the sets, read off an identity X,
    are the reference's."""
    rng = np.random.default_rng(3)
    n, deg = 1500, 40
    rows = np.repeat(np.arange(n), deg)
    A = sp.csr_matrix((np.ones(n * deg, np.float32), (rows, rng.integers(0, n, n * deg))), shape=(n, n))
    X = sp.identity(n, dtype=np.float32, format="csr")
    got, nnz = _niche.niche_aggregate(A, X, "mean", 3)
    expect, expect_nnz = niche_ref.cellcharter(A, X, 3, "mean")
    assert list(nnz) == expect_nnz
    for k, H in enumerate(niche_ref.hops(A, 3)):
        np.testing.assert_array_equal(got[:, (k + 1) * n:(k + 2) * n] != 0, H.toarray() != 0)
    np.testing.assert_array_equal(got, expect)


@pytest.mark.parametrize("layout", ["csr", "csc"])
@pytest.mark.parametrize("index_dtype", ["int32", "int64"])
def test_device_graph_and_x_equal_host(layout, index_dtype):
    import torch

    A = GRAPHS["noncanonical"] if layout == "csr" else GRAPHS["csc"]
    adata = make_adata(A)
    codes, C = _codes(adata)
    idt = getattr(torch, index_dtype)
    if layout == "csr":
        dA = torch.sparse_csr_tensor(torch.from_numpy(A.indptr).to(idt), torch.from_numpy(A.indices).to(idt), torch.from_numpy(A.data),
                                     size=A.shape, device="cuda")
    else:
        dA = torch.sparse_csc_tensor(torch.from_numpy(A.indptr).to(idt), torch.from_numpy(A.indices).to(idt), torch.from_numpy(A.data),
                                     size=A.shape, device="cuda")
    np.testing.assert_array_equal(_niche.niche_profile(dA, codes, C, 3), _niche.niche_profile(A, codes, C, 3))
    Xh = adata.X
    Xd_dense = torch.from_numpy(Xh.toarray()).cuda()
    Xd_csr = torch.sparse_csr_tensor(torch.from_numpy(Xh.indptr).to(idt), torch.from_numpy(Xh.indices).to(idt), torch.from_numpy(Xh.data),
                                     size=Xh.shape, device="cuda")
    for mode, dist in (("utag", 1), ("mean", 3), ("variance", 2)):
        host, host_nnz = _niche.niche_aggregate(A, Xh, mode, dist)
        for Xd in ((Xd_dense, Xd_csr) if mode != "variance" else (Xd_csr,)):
            for g in (A, dA):
                got, nnz = _niche.niche_aggregate(g, Xd, mode, dist)
                np.testing.assert_array_equal(got, host)
                np.testing.assert_array_equal(nnz, host_nnz)
    # the public functions take device graphs and X
    standin.install()
    a_host = make_adata(A)
    _niche.calculate_niche_utag(a_host, 0.5)
    host_calls = list(standin.CALLS)
    standin.install()
    a_dev = make_adata(A)
    a_dev.obsp["spatial_connectivities"], a_dev.X = dA, Xd_csr
    _niche.calculate_niche_utag(a_dev, 0.5)
    for (n1, x1, _), (n2, x2, _) in zip(host_calls, standin.CALLS):
        assert n1 == n2
        np.testing.assert_array_equal(x1, x2)
    np.testing.assert_array_equal(a_host.obs["utag_niche_res=0.5"].to_numpy(), a_dev.obs["utag_niche_res=0.5"].to_numpy())


def test_empty_graph():
    n = 50
    A = sp.csr_matrix((n, n), dtype=np.float32)
    adata = make_adata(A)
    codes, C = _codes(adata)
    np.testing.assert_array_equal(_niche.niche_profile(A, codes, C, 3), np.zeros((n, C)))
    out, _ = _niche.niche_aggregate(A, adata.X, "utag")
    np.testing.assert_array_equal(out, niche_ref.utag(A, adata.X))
    out, nnz = _niche.niche_aggregate(A, adata.X, "mean", 3)
    expect, expect_nnz = niche_ref.cellcharter(A, adata.X, 3, "mean")
    np.testing.assert_array_equal(out, expect)
    assert list(nnz) == expect_nnz


def test_profile_one_million_spots():
    A = synth.hex_graph(1000, 1000)
    rng = np.random.default_rng(7)
    codes = rng.integers(0, 20, A.shape[0]).astype(np.int32)
    got = _niche.niche_profile(A, codes, 20, 3, [1.0, 0.5, 0.25])
    np.testing.assert_array_equal(got, niche_ref.profile(A, codes, 20, 3, [1.0, 0.5, 0.25]))


def test_cellcharter_200k_cells():
    A = synth.hex_graph(400, 500)
    n, m = A.shape[0], 300
    X = sp.random(n, m, density=0.1, format="csr", dtype=np.float32, random_state=5)
    X.data = np.floor(X.data * 8).astype(np.float32)
    got, nnz = _niche.niche_aggregate(A, X, "mean", 3)
    expect, expect_nnz = niche_ref.cellcharter(A, X, 3, "mean")
    assert list(nnz) == expect_nnz
    np.testing.assert_array_equal(got, expect)


def test_boolean_device_graph_refused():
    import torch

    A = GRAPHS["hex"]
    dA = torch.sparse_csr_tensor(torch.from_numpy(A.indptr.astype(np.int64)), torch.from_numpy(A.indices.astype(np.int64)),
                                 torch.ones(A.nnz, dtype=torch.bool), size=A.shape, device="cuda")
    with pytest.raises(TypeError, match="Boolean connectivity graphs"):
        _niche.niche_profile(dA, np.zeros(A.shape[0], np.int32), 1, 2)
    # a column index out of range, in the canonical (profile) and the stored (UTAG) order
    bad = torch.sparse_csr_tensor(torch.tensor([0, 1, 1]), torch.tensor([5]), torch.tensor([1.0]), size=(2, 2)).cuda()
    with pytest.raises(ValueError, match="out of range"):
        _niche.niche_profile(bad, np.zeros(2, np.int32), 1)
    with pytest.raises(ValueError, match="out of range"):
        _niche.niche_aggregate(bad, np.ones((2, 3)), "utag")


def test_cellcharter_knn15_long_rows():
    """A kNN graph with 15 neighbours at distance 3: hop-3 bounds in the thousands, so most rows use global-memory tables,
    batched under the memory budget.  Equal to the restatement."""
    from sklearn.neighbors import NearestNeighbors

    xy = np.random.default_rng(11).random((100_000, 2))
    A = NearestNeighbors(n_neighbors=15).fit(xy).kneighbors_graph(mode="connectivity").tocsr().astype(np.float32)
    X = sp.random(A.shape[0], 6, density=0.3, format="csr", dtype=np.float32, random_state=2)
    got, nnz = _niche.niche_aggregate(A, X, "mean", 3)
    expect, expect_nnz = niche_ref.cellcharter(A, X, 3, "mean")
    assert list(nnz) == expect_nnz
    np.testing.assert_array_equal(got, expect)

