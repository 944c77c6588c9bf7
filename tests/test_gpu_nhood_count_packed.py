"""GPU parity of the row-record count kernel, which covers 64 permutations per warp (two per lane, counters packed as the
16-bit halves of one word) from the group-major label matrix [PB/64][N+1][64].

Permutation counts around the group edges (P = 1 ... 65, 1000), u8 and u16 labels, symmetric / directed graphs with self
loops, library segments (the transpose scatters rows through `order`), the CSR-row cross-check (count_sym = 0) and the fast
RNG mode are compared with the oracle.  The overflow rule of the 16-bit halves is exercised with cases that put more than
65 536 increments of one bin and permutation into one CTA's chunk; `recs_rule` restates the launch rule so that each case
asserts which side of it it is on."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import NhoodPlan
from tests import philox_ref
from tools import synth

pytestmark = pytest.mark.gpu

RECS_NO_DRAIN = 65535 // 3  # a chunk of at most this many records cannot carry a 16-bit half


def recs_rule(n_recs: int, P: int, sm_count: int) -> tuple[int, bool]:
    """(records per CTA, drains between rounds) of ``launch_count``'s record-kernel grid (nhood.cu):

        rgroups = ceil(P / 64); pchunk = (4 * sm + rgroups / 2) / rgroups, or the first q in [pchunk, 2 pchunk] with
        q * rgroups % sm == 0; pchunk <= ceil(n_recs / 1024); recs_per_cta = ceil(n_recs / pchunk);
        drain iff recs_per_cta > 65535 / 3.
    """
    rgroups = -(-P // 64)
    pchunk = max((4 * sm_count + rgroups // 2) // rgroups, 1)
    for q in range(pchunk, 2 * pchunk + 1):
        if q * rgroups % sm_count == 0:
            pchunk = q
            break
    pchunk = max(min(pchunk, -(-n_recs // 1024)), 1)
    recs_per_cta = -(-n_recs // pchunk)
    return recs_per_cta, recs_per_cta > RECS_NO_DRAIN


def n_records(g: sp.csr_matrix, symmetric: bool) -> int:
    a = sp.triu(g, format="csr") if symmetric else g
    return int(((np.diff(a.indptr) + 2) // 3).sum())


def _sym_selfloops(n: int, seed: int) -> sp.csr_matrix:
    rng = np.random.default_rng(seed)
    a = sp.random(n, n, density=4.0 / n, format="csr", random_state=seed, dtype=np.float32)
    g = (((a + a.T) > 0).astype(np.float32) + sp.diags((rng.random(n) < 0.3).astype(np.float32))).tocsr()
    g.eliminate_zeros()
    g.sort_indices()
    return g


def _graph(kind: str) -> sp.csr_matrix:
    if kind == "hex":
        return synth.hex_graph(37, 41)
    if kind == "sym_selfloops":
        return _sym_selfloops(1700, 4)
    return synth.knn_graph(np.random.default_rng(9).random((1500, 2)), 6)  # directed


@pytest.mark.parametrize("P", [1, 31, 32, 33, 63, 64, 65, 1000])
@pytest.mark.parametrize("kind", ["hex", "sym_selfloops", "knn_directed"])
def test_perm_counts_around_group_edges(kind, P):
    g = _graph(kind)
    n_cls = 13
    base = np.random.default_rng(P).integers(0, n_cls, g.shape[0]).astype(np.uint32)
    st = spawn_states(100 + P, P)
    exp = ref.nhood_perm_counts(g.indptr, g.indices, base, n_cls, st)
    plan = NhoodPlan(g.indptr, g.indices, n_cls)
    plan.set_base(base)
    np.testing.assert_array_equal(plan.permute(st), exp)
    plan.set_option("count_sym", 0)  # the CSR-row kernel reads the same label matrix
    np.testing.assert_array_equal(plan.permute(st), exp)
    plan.close()


@pytest.mark.parametrize("n_cls", [30, 45, 300])
@pytest.mark.parametrize("P", [33, 65])
def test_label_widths_and_histogram_layouts(n_cls, P):
    """30: record kernel; 45: CSR-row kernel with 16 permutations per CTA; 300: u16 labels and global atomics."""
    g = _sym_selfloops(1200, n_cls)
    base = np.random.default_rng(n_cls).integers(0, n_cls, g.shape[0]).astype(np.uint32)
    st = spawn_states(7 * n_cls, P)
    plan = NhoodPlan(g.indptr, g.indices, n_cls)
    plan.set_base(base)
    np.testing.assert_array_equal(plan.permute(st), ref.nhood_perm_counts(g.indptr, g.indices, base, n_cls, st))
    plan.close()


@pytest.mark.parametrize("n_cls", [11, 300])
@pytest.mark.parametrize("kind", ["hex", "knn_directed"])
def test_library_key_scatter(kind, n_cls):
    g = _graph(kind)
    n = g.shape[0]
    rng = np.random.default_rng(3)
    base = rng.integers(0, n_cls, n).astype(np.uint32)
    lib = rng.integers(0, 3, n).astype(np.int32)
    P = 70
    st = spawn_states(21, P)
    plan = NhoodPlan(g.indptr, g.indices, n_cls)
    plan.set_base(base, lib, 3)
    exp = ref.nhood_perm_counts(g.indptr, g.indices, base, n_cls, st, lib, 3)
    np.testing.assert_array_equal(plan.permute(st), exp)
    plan.close()


@pytest.mark.parametrize("P", [1, 63, 65, 130])
@pytest.mark.parametrize("kind", ["sym_selfloops", "knn_directed"])
def test_philox_counts(kind, P):
    g = _graph(kind)
    n_cls = 9
    base = np.random.default_rng(P).integers(0, n_cls, g.shape[0]).astype(np.uint32)
    lib = (np.arange(g.shape[0]) % 2).astype(np.int32)
    plan = NhoodPlan(g.indptr, g.indices, n_cls)
    plan.set_base(base, lib, 2)
    plan.upload_philox(11, 5, P)
    labs = plan.shuffled_labels(0, P)
    np.testing.assert_array_equal(labs, philox_ref.philox_labels(base, 11, range(5, 5 + P), lib, 2))
    plan.run_async()
    got = plan.download()
    for p in range(P):
        np.testing.assert_array_equal(got[p], ref.nhood_count(g.indptr, g.indices, labs[p], n_cls))
    plan.close()


def _sm_count() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("kind", ["hex", "knn_directed"])
def test_overflow_rule_single_class(kind):
    """Every label equal: every increment of a CTA lands on one bin of each permutation, far more than a 16-bit half holds."""
    P = 10000
    if kind == "hex":
        g, symmetric = synth.hex_graph(400, 500), True
    else:
        g, symmetric = synth.knn_graph(np.random.default_rng(1).random((100_000, 2)), 6), False
    recs_per_cta, drains = recs_rule(n_records(g, symmetric), P, _sm_count())
    assert drains and 3 * recs_per_cta > 65535, recs_per_cta
    plan = NhoodPlan(g.indptr, g.indices, 2)
    plan.set_option("perm_chunk", P)  # one launch for all permutations: the grid the rule above describes
    plan.set_base(np.zeros(g.shape[0], np.uint32))
    plan.upload_philox(3, 0, P)
    plan.run_async()
    got = plan.download().reshape(P, 4)
    assert (got[:, 0] == g.nnz).all() and (got[:, 1:] == 0).all()
    plan.close()


def test_overflow_rule_mixed_labels():
    """One class holds 95 % of the labels: the drained bin and the bins that never reach 2^15 both stay exact."""
    P = 10000
    g = synth.knn_graph(np.random.default_rng(2).random((100_000, 2)), 6)
    recs_per_cta, drains = recs_rule(n_records(g, False), P, _sm_count())
    assert drains, recs_per_cta
    rng = np.random.default_rng(8)
    base = np.where(rng.random(g.shape[0]) < 0.95, 0, rng.integers(1, 4, g.shape[0])).astype(np.uint32)
    plan = NhoodPlan(g.indptr, g.indices, 4)
    plan.set_option("perm_chunk", P)
    plan.set_base(base)
    plan.upload_philox(5, 0, P)
    plan.run_async()
    got = plan.download()
    assert (got.reshape(P, -1).sum(axis=1, dtype=np.int64) == g.nnz).all()
    for p in (0, 1, 62, 63, 64, 5001, P - 1):
        labs = plan.shuffled_labels(p, p + 1)[0]
        np.testing.assert_array_equal(got[p], ref.nhood_count(g.indptr, g.indices, labs, 4))
    plan.close()


def test_rule_sides_at_benchmark_shapes():
    """On 132 SMs a 1M-spot hex graph x 1000 permutations and 300 K directed kNN x 4416 permutations drain; 100 K records x
    1000 permutations run in one round."""
    assert recs_rule(999_999, 1000, 132) == (30303, True)
    assert recs_rule(600_000, 4416, 132)[1]
    assert not recs_rule(100_000, 1000, 132)[1]
