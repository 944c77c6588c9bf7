"""The post-processors and ``GraphBuilderCSR.combine`` on device graphs against the host path on scipy copies of the same
matrices, at the inputs where the device steps differ in kind from scipy / numpy:

* non-finite and signed-zero distances (NaN of either sign, all-NaN rows, +inf as the maximum and at interior order
  statistics, stored -0.0 and +0.0, rows left empty) through every percentile of {0, 37.5, 50, 90, 100} and the interval, each
  alone and followed by every transform, in float32 and float64;
* non-finite connectivities through the transforms (sklearn's cosine refuses them, spectral carries them);
* weighted spectral on columns of high in-degree, whose float32 column sums depend on the order they are added in, run twice;
* graphs of a million points built on the device: kNN(6), a radius graph with more than 2^24 float32 distances, the
  ``n_rings=3`` hex lattice, and 20 interleaved libraries combined.

"Equal" is ``assert_same_csr``: the same indptr, indices and values bit for bit, explicit zeros included.  Where the host
raises, the device raises the same exception type.  The percentile arithmetic itself is pinned on the CPU by
``tests/test_graph_percentile_spec.py``."""

from __future__ import annotations

import warnings

import numpy as np
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

from squidpy_b200._constants import Transform  # noqa: E402
from squidpy_b200.gr import GridBuilder, KNNBuilder, RadiusBuilder  # noqa: E402
from squidpy_b200.gr import neighbors as nb  # noqa: E402
from tests.test_gpu_graph_postprocess import to_dev, to_host  # noqa: E402
from tests.test_neighbors_api_host import assert_same_csr  # noqa: E402
from tools import synth  # noqa: E402

pytestmark = pytest.mark.gpu

NEG_NAN = np.array(0xFFF8000000000000, np.uint64).view(np.float64)[()]  # a NaN with its sign bit set
PCT, INTERVAL = [0.0, 37.5, 50.0, 90.0, 100.0], (0.5, 3.0)
TRANSFORMS = [None, Transform.NONE, Transform.SPECTRAL, Transform.COSINE]


def run(steps, adj, dst):
    for s in steps:
        adj, dst = s(adj, dst)
    return adj, dst


def host_run(steps, adj, dst):
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        return run(steps, adj.copy(), dst.copy())


def canonical_nan(m: sp.csr_matrix) -> sp.csr_matrix:
    """NaN values replaced by one NaN: x86 and the GPU produce NaNs with different bit patterns (0 * inf, inf - inf)."""
    m = m.copy()
    m.data[np.isnan(m.data)] = np.nan
    return m


def check_steps(steps, adj: sp.csr_matrix, dst: sp.csr_matrix, nan_payloads: bool = True) -> None:
    """The steps on device copies of (adj, dst) equal the host path on scipy copies, or raise the host's exception type.
    nan_payloads=False compares the connectivities with every NaN made one (values computed from non-finite inputs)."""
    try:
        want = host_run(steps, adj, dst)
    except Exception as e:  # noqa: BLE001 - whatever the host raises, the device must raise too
        with pytest.raises(type(e)):
            run(steps, to_dev(adj), to_dev(dst))
        return
    got = [to_host(t) for t in run(steps, to_dev(adj), to_dev(dst))]
    if not nan_payloads:
        got[0], want = canonical_nan(got[0]), (canonical_nan(want[0]), want[1])
    assert_same_csr(got[0], want[0])
    assert_same_csr(got[1], want[1])


# ---- non-finite and signed-zero distances -------------------------------------------------------------------------------
def base_graph(n: int = 60, seed: int = 0) -> tuple[sp.csr_matrix, sp.csr_matrix]:
    """Connectivities of ones and distances in [0.25, 4) with ties, rows of 0 to 11 entries (some with the diagonal);
    row 3 stores nothing."""
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for i in range(n):
        k = 0 if i == 3 else int(rng.integers(1, 12))
        c = np.sort(rng.choice(n, k, replace=False))
        rows += [i] * k
        cols += c.tolist()
    d = np.round(rng.uniform(0.25, 4.0, len(rows)), 1)  # ties
    dst = sp.csr_matrix((d, (rows, cols)), shape=(n, n))
    adj = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n, n))
    return adj, dst


def _row(dst, i):
    return slice(dst.indptr[i], dst.indptr[i + 1])


def edge_case(name: str, dtype) -> tuple[sp.csr_matrix, sp.csr_matrix]:
    adj, dst = base_graph()
    v = dst.data
    rng = np.random.default_rng(1)
    if name == "nan":
        v[17] = np.nan
    elif name == "neg_nan":
        v[17] = NEG_NAN
    elif name == "nan_row":
        v[_row(dst, 5)] = np.nan
    elif name == "inf_max":
        v[17] = np.inf
    elif name == "inf_interior":  # 60 % infinite: the order statistics above q = 40 are infinite
        v[rng.random(v.size) < 0.6] = np.inf
    elif name == "signed_zeros":
        r = rng.random(v.size)
        v[r < 0.3] = -0.0
        v[(r >= 0.3) & (r < 0.5)] = 0.0
    elif name == "empty_rows":  # row 3 stores nothing; row 7's distances exceed every threshold but q = 100's and the interval
        v[_row(dst, 7)] = 1e6
    dst = dst.astype(dtype)
    if name == "neg_nan":
        assert np.isnan(dst.data[17]) and np.signbit(dst.data[17])
    return adj, dst


EDGE_CASES = ["finite", "nan", "neg_nan", "nan_row", "inf_max", "inf_interior", "signed_zeros", "empty_rows"]
PRUNERS = [f"percentile_{q}" for q in PCT] + ["interval"]


def pruner(name: str):
    return nb.DistanceIntervalPostprocessor(INTERVAL) if name == "interval" else nb.PercentilePostprocessor(float(name.split("_")[1]))


@pytest.mark.parametrize("dtype", [np.float32, np.float64], ids=["float32", "float64"])
@pytest.mark.parametrize("prune", PRUNERS)
@pytest.mark.parametrize("case", EDGE_CASES)
def test_distances_with_non_finite_and_signed_zero_values(case, prune, dtype):
    adj, dst = edge_case(case, dtype)
    for t in TRANSFORMS:
        steps = [pruner(prune)] + ([] if t is None else [nb.TransformPostprocessor(t)])
        check_steps(steps, adj, dst)


def test_nan_distance_prunes_nothing_and_q100_over_inf_is_accepted():
    # the host's threshold is NaN in both cases; `dst > nan` marks nothing
    for case, q in (("nan", 50.0), ("neg_nan", 0.0), ("inf_max", 100.0)):
        adj, dst = edge_case(case, np.float32)
        a, d = (to_host(t) for t in nb.PercentilePostprocessor(q)(to_dev(adj), to_dev(dst)))
        assert_same_csr(a, adj)
        assert_same_csr(d, dst)


# ---- non-finite connectivities ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value", ["nan", "neg_nan", "inf", "neg_inf", "nan_row"])
def test_non_finite_connectivities_through_the_transforms(value):
    adj, dst = base_graph(seed=2)
    adj.data[:] = np.random.default_rng(3).uniform(0.1, 2.0, adj.nnz).astype(np.float32)
    if value == "nan_row":
        adj.data[_row(adj, 5)] = np.nan
    else:
        adj.data[17] = {"nan": np.nan, "neg_nan": NEG_NAN, "inf": np.inf, "neg_inf": -np.inf}[value]
    for steps in ([nb.TransformPostprocessor(Transform.COSINE)], [nb.TransformPostprocessor(Transform.SPECTRAL)],
                  [nb.TransformPostprocessor(Transform.NONE)], [nb.PercentilePostprocessor(50.0), nb.TransformPostprocessor(Transform.COSINE)]):
        check_steps(steps, adj, dst, nan_payloads=False)
    with pytest.raises(ValueError, match="NaN" if "nan" in value else "infinity"):
        nb.TransformPostprocessor(Transform.COSINE)(to_dev(adj), to_dev(dst))


# ---- weighted spectral --------------------------------------------------------------------------------------------------
def _weights(rng, m: int) -> np.ndarray:
    return rng.uniform(0.05, 1.0, m).astype(np.float32)  # full float32 mantissas: no column sums exactly


def radius_graph() -> tuple[sp.csr_matrix, sp.csr_matrix]:
    from sklearn.neighbors import radius_neighbors_graph

    rng = np.random.default_rng(4)
    dst = radius_neighbors_graph(rng.uniform(0.0, 1.0, (3000, 2)), 0.18, mode="distance").tocsr()  # about 300 per row
    dst.sort_indices()
    adj = sp.csr_matrix((_weights(rng, dst.nnz), dst.indices.copy(), dst.indptr.copy()), shape=dst.shape)
    return adj, dst


def star_graph(n: int = 200_001) -> tuple[sp.csr_matrix, sp.csr_matrix]:
    rng = np.random.default_rng(5)
    rows = np.concatenate([np.zeros(n - 1, np.int64), np.arange(1, n)])
    cols = np.concatenate([np.arange(1, n), np.zeros(n - 1, np.int64)])
    dst = sp.csr_matrix((rng.uniform(0.5, 2.0, rows.size), (rows, cols)), shape=(n, n))
    adj = sp.csr_matrix((_weights(rng, dst.nnz), dst.indices.copy(), dst.indptr.copy()), shape=dst.shape)
    return adj, dst


@pytest.mark.parametrize("graph", ["radius", "star"])
def test_weighted_spectral_equals_host_and_repeats(graph):
    adj, dst = radius_graph() if graph == "radius" else star_graph()
    # the inputs discriminate: float64 column sums rounded to float32 differ from scipy's float32 sums somewhere
    f32 = np.asarray(adj.sum(axis=0)).ravel()
    assert (np.asarray(adj.sum(axis=0, dtype=np.float64)).ravel().astype(np.float32) != f32).any()
    step = nb.TransformPostprocessor(Transform.SPECTRAL)
    ha, hd = host_run([step], adj, dst)
    first = None
    for _ in range(3):
        a, d = (to_host(t) for t in step(to_dev(adj), to_dev(dst)))
        assert_same_csr(a, ha)
        assert_same_csr(d, hd)
        if first is not None:
            assert_same_csr(a, first)
        first = a


# ---- size ---------------------------------------------------------------------------------------------------------------
def check_device_graph(steps, adj, dst) -> None:
    """The steps on a graph built on the device equal the host path on scipy copies of it."""
    ha, hd = to_host(adj), to_host(dst)
    want = host_run(steps, ha, hd)
    got = run(steps, adj, dst)
    assert_same_csr(to_host(got[0]), want[0])
    assert_same_csr(to_host(got[1]), want[1])


def test_knn_of_a_million_points_percentile_then_cosine():
    co = np.random.default_rng(6).uniform(0.0, 1000.0, (1_000_000, 2))
    adj, dst = KNNBuilder(n_neighs=6).build(torch.tensor(co, device="cuda"))
    check_device_graph([nb.PercentilePostprocessor(90.0), nb.TransformPostprocessor(Transform.COSINE)], adj, dst)


def test_radius_graph_with_more_than_2_24_float32_distances():
    co = np.random.default_rng(7).uniform(0.0, 1000.0, (1_000_000, 2))
    adj, dst = RadiusBuilder(radius=2.6).build(torch.tensor(co, device="cuda"))  # mean degree about 21
    dst = torch.sparse_csr_tensor(dst.crow_indices(), dst.col_indices(), dst.values().float(), size=dst.shape)
    assert dst.values().numel() > 2**24
    for q in (90.0, 99.99):
        check_device_graph([nb.PercentilePostprocessor(q)], adj, dst)
    check_device_graph([nb.PercentilePostprocessor(50.0), nb.TransformPostprocessor(Transform.COSINE)], adj, dst)


def test_grid_n_rings_3_on_the_million_spot_lattice():
    adj, dst = GridBuilder(6, n_rings=3).build(torch.tensor(synth.hex_coords(1000, 1000), device="cuda"))
    check_device_graph([nb.PercentilePostprocessor(60.0), nb.TransformPostprocessor(Transform.SPECTRAL)], adj, dst)


def test_combine_of_20_interleaved_libraries():
    rng = np.random.default_rng(8)
    n, n_libs = 1_000_000, 20
    co = rng.uniform(0.0, 1000.0, (n, 2))
    lib = rng.integers(0, n_libs, n)
    blocks, host_blocks, ixs = [], [], []
    for b in range(n_libs):
        ix = rng.permutation(np.flatnonzero(lib == b))  # a block's rows map out of order: the rows are re-sorted after the scatter
        a, d = KNNBuilder(n_neighs=6).build(torch.tensor(co[ix], device="cuda"))
        blocks.append((a, d))
        host_blocks.append((to_host(a), to_host(d)))
        ixs.append(ix)
    ixs = np.concatenate(ixs).tolist()
    adj, dst = KNNBuilder().combine(blocks, ixs)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", sp.SparseEfficiencyWarning)
        ha, hd = KNNBuilder().combine(host_blocks, ixs)
    assert_same_csr(to_host(adj), ha)
    assert_same_csr(to_host(dst), hd)
