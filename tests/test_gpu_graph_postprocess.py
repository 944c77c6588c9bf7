"""The public post-processors and ``GraphBuilderCSR.combine`` on device graphs: every golden case of
``tests/golden/postprocessors.npz`` (the unmodified reference on host copies) run on the GPU, from torch ``sparse_csr`` tensors
with int32 and int64 indices and from cupyx-style CSRs; spectral, weighted too, against the host path; the refusals, each
leaving the context usable."""

from __future__ import annotations

import builtins
import json
import warnings

import numpy as np
import pytest
import scipy.sparse as sp

torch = pytest.importorskip("torch")

from squidpy_b200._constants import Transform  # noqa: E402
from squidpy_b200.gr import neighbors as nb  # noqa: E402
from tests.test_neighbors_api_host import GOLD, assert_same_csr, combine_blocks, gold_csr, make_step  # noqa: E402

pytestmark = pytest.mark.gpu


def to_dev(m: sp.csr_matrix, index_dtype=torch.int32):
    return torch.sparse_csr_tensor(torch.tensor(m.indptr, dtype=index_dtype), torch.tensor(m.indices, dtype=index_dtype), torch.tensor(m.data),
                                   size=m.shape).cuda()


class CupyxCsr:
    """A cupyx-style CSR: ``format``, ``shape`` and ``indptr`` / ``indices`` / ``data`` exposing the CUDA Array Interface."""

    format = "csr"

    def __init__(self, t):
        self.shape = tuple(t.shape)
        self.indptr, self.indices, self.data = t.crow_indices(), t.col_indices(), t.values()


def to_host(t) -> sp.csr_matrix:
    assert t.layout == torch.sparse_csr and t.is_cuda
    assert t.crow_indices().dtype == torch.int32 and t.col_indices().dtype == torch.int32
    c = t.cpu()
    idx = c.col_indices().numpy()
    ptr = c.crow_indices().numpy()
    assert all((np.diff(idx[ptr[i]:ptr[i + 1]]) > 0).all() for i in range(len(ptr) - 1)), "columns must ascend in every row"
    return sp.csr_matrix((c.values().numpy(), idx, ptr), shape=tuple(t.shape))


VARIANTS = {"i32": lambda m: to_dev(m), "i64": lambda m: to_dev(m, torch.int64), "cupyx": lambda m: CupyxCsr(to_dev(m))}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", [str(n) for n in GOLD["pp_cases"]])
def test_device_postprocessors_equal_reference(name, variant):
    adj, dst = (VARIANTS[variant](gold_csr(f"pp/{name}/{k}_in")) for k in ("adj", "dst"))
    steps = json.loads(str(GOLD[f"pp/{name}/steps"]))
    if f"pp/{name}/error" in GOLD:
        with pytest.raises(getattr(builtins, str(GOLD[f"pp/{name}/error"]))):
            for step in steps:
                adj, dst = make_step(step)(adj, dst)
        return
    for step in steps:
        adj, dst = make_step(step)(adj, dst)
    assert_same_csr(to_host(adj), gold_csr(f"pp/{name}/adj_out"))
    assert_same_csr(to_host(dst), gold_csr(f"pp/{name}/dst_out"))


@pytest.mark.parametrize("name", [str(n) for n in GOLD["combine_cases"]])
def test_device_combine_equals_reference(name):
    blocks, ixs = combine_blocks(name)
    adj, dst = nb.KNNBuilder().combine([(to_dev(a), to_dev(d)) for a, d in blocks], ixs)
    assert_same_csr(to_host(adj), gold_csr(f"combine/{name}/adj_out"))
    assert_same_csr(to_host(dst), gold_csr(f"combine/{name}/dst_out"))


@pytest.mark.parametrize("name", ["weighted_float32_none", "chain3_float64", "diff_float64_pct50", "same_float32_interval_zeros_empty"])
def test_device_spectral(name):
    adj, dst = gold_csr(f"pp/{name}/adj_in"), gold_csr(f"pp/{name}/dst_in")
    da, dd = nb.TransformPostprocessor(Transform.SPECTRAL)(to_dev(adj), to_dev(dst))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        ha, hd = nb.TransformPostprocessor(Transform.SPECTRAL)(adj.copy(), dst.copy())
    assert_same_csr(to_host(dd), hd)
    assert_same_csr(to_host(da), ha)  # weighted too: the column sums are scipy's float32 sums in row order


def test_device_results_equal_host_results_on_a_knn_graph():
    rng = np.random.default_rng(3)
    co = rng.uniform(0, 1000, (5000, 2))
    adj, dst = nb.KNNBuilder(n_neighs=6).build(torch.tensor(co, device="cuda"))
    hadj, hdst = nb.KNNBuilder(n_neighs=6).build(co)
    for steps in ([nb.PercentilePostprocessor(60.0), nb.TransformPostprocessor(Transform.COSINE)],
                  [nb.DistanceIntervalPostprocessor((5.0, 15.0)), nb.TransformPostprocessor(Transform.SPECTRAL)]):
        a, d, ha, hd = adj, dst, hadj.copy(), hdst.copy()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", sp.SparseEfficiencyWarning)
            for s in steps:
                a, d = s(a, d)
                ha, hd = s(ha, hd)
        assert_same_csr(to_host(a), ha)
        assert_same_csr(to_host(d), hd)


def test_refusals_leave_the_context_usable():
    adj, dst = gold_csr("pp/same_float64_interval/adj_in"), gold_csr("pp/same_float64_interval/dst_in")
    pct = nb.PercentilePostprocessor(50.0)
    with pytest.raises(TypeError, match="float32"):
        pct(to_dev(adj.astype(np.float64)), to_dev(dst))
    with pytest.raises(TypeError, match="float32 or float64"):
        pct(to_dev(adj), to_dev(dst.astype(np.int32)))
    with pytest.raises(TypeError, match="one on the host"):
        pct(adj, to_dev(dst))
    bad = dst.copy()
    r = int(np.argmax(np.diff(bad.indptr) >= 2))
    s0 = bad.indptr[r]
    bad.indices[s0], bad.indices[s0 + 1] = bad.indices[s0 + 1], bad.indices[s0]
    with pytest.raises(ValueError, match="strictly increasing"):
        pct(to_dev(adj), to_dev(bad))
    neg = dst.copy()
    neg.data[:] = -1.0
    with pytest.raises(NotImplementedError, match="threshold"):
        pct(to_dev(adj), to_dev(neg))
    with pytest.raises(IndexError):
        pct(to_dev(adj), to_dev(sp.csr_matrix(dst.shape, dtype=np.float64)))
    with pytest.raises(ValueError, match="permutation|distinct"):
        nb.KNNBuilder().combine([(to_dev(adj), to_dev(dst))], [0] * adj.shape[0])
    a, d = pct(to_dev(adj), to_dev(dst))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", sp.SparseEfficiencyWarning)
        ha, hd = pct(adj.copy(), dst.copy())
    assert_same_csr(to_host(a), ha)
    assert_same_csr(to_host(d), hd)
