"""GPU parity of the ligrec permutation counts on the paths the small cases never take: many clusters (the group-mean
kernel's opt-in shared memory), several permutation chunks, and labels shuffled by the list replay (shuffle_algo 7) and the
region replay (shuffle_algo 9).

Expression is integer-valued (Poisson), so every float64 group sum is exact in any order.  That makes a fast exact
reference possible at large shapes: shuffle the labels with the oracle's numpy-stream replay, form the group sums with one
``bincount`` per gene over ``p * C + label``, multiply by ``inv_counts`` and count ``shuf > obs``.  With integer data exact
ties ``shuf == obs`` are common, so the cases also pin the strict ``>``."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pandas as pd
import pytest

from oracle import ref
from squidpy_b200._lib import check, default_context, load
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import ligrec_analysis
from tests.device_attrs import H100_SMEM_OPTIN, smem_optin

pytestmark = pytest.mark.gpu


def group_means_smem(n_cls: int) -> int:
    """Dynamic shared memory of ``ligrec_group_means_kernel`` (nhood.cu §6): ``smem = 4 * C * 32 * sizeof(double)``.
    Above 48 KB the launch needs the opt-in attribute; ``smem <= c->smem_optin`` is required."""
    return 4 * n_cls * 32 * 8


def perm_chunks(n_perms: int, upload_chunk: int, n_cls: int, n_genes: int) -> list[int]:
    """Permutations per pass of ``sqb_ligrec_counts``: ``chunk = min(h->chunk, 2^30 / (C * G * 8))`` (at least 1)."""
    gcap = (1 << 30) // (n_cls * n_genes * 8)
    chunk = min(upload_chunk, max(gcap, 1))
    return [min(chunk, n_perms - p0) for p0 in range(0, n_perms, chunk)]


def upload_chunk(n_perms: int, perm_chunk: int = 0, stride: int = 0) -> int:
    """``h->chunk`` after ``sqb_nhood_permute_upload`` (nhood.cu ``auto_chunk``): ``perm_chunk`` rounded up to 32, else
    ~8 GB / (6 * stride) clamped to [32, 16384] and rounded down to 32; never more than ``n_perms`` rounded up to 32."""
    if perm_chunk > 0:
        ch = (perm_chunk + 31) // 32 * 32
    else:
        ch = min(max(int(8e9) // (6 * stride), 32), 16384) // 32 * 32
    return min(ch, (n_perms + 31) // 32 * 32)


def auto_replay(n: int, np_chunk: int, sm_count: int) -> int:
    """The exact replay auto mode picks for a chunk of ``np_chunk`` permutations of ``n`` labels (nhood.cu
    ``part_replay_shape`` and ``launch_shuffle``): ``np > 2 * sm_count && n >= 524288`` -> 9 (region replay, when every
    segment fits its region limits), ``np > 2 * sm_count && n >= 65536`` -> 7 (list replay), otherwise 1 (one CTA per
    permutation) or 2 (one warp per permutation)."""
    if np_chunk > 2 * sm_count:
        return 9 if n >= 524288 else 7 if n >= 65536 else 2
    return 1


def make_case(seed, n_cells, n_genes, n_cls, n_inter, lam=0.6):
    rng = np.random.default_rng(seed)
    x = rng.poisson(lam, size=(n_cells, n_genes)).astype(np.float64)
    cl = rng.integers(0, n_cls, n_cells)
    cl[:n_cls] = np.arange(n_cls)  # every cluster present
    inter = np.unique(np.stack([rng.integers(0, n_genes, n_inter), rng.integers(0, n_genes, n_inter)], 1), axis=0)
    return x, cl, inter


def fast_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid, batch=64):
    """``ref.ligrec_counts`` for integer-valued ``x``: the group sums are exact, so their order does not matter.  Returns
    (counts of shuf > obs, number of exact ties shuf == obs among the valid entries)."""
    n = x.shape[0]
    a, b = cpairs[:, 0], cpairs[:, 1]
    obs = mean_obs[a][:, inter[:, 0]].T + mean_obs[b][:, inter[:, 1]].T
    genes, pos = np.unique(inter, return_inverse=True)  # only the genes that take part in an interaction
    rec, lig = pos.reshape(inter.shape).T
    counts = np.zeros(obs.shape, np.int64)
    ties = 0
    sub = max(1, 4_000_000 // obs.size)  # permutations compared at once
    for p0 in range(0, states.shape[0], batch):
        labs = ref.shuffle_labels(np.asarray(cl, np.uint32), states[p0 : p0 + batch]).astype(np.int64)
        assert labs.shape[1] == n
        nb = labs.shape[0]
        key = (labs + (np.arange(nb) * n_cls)[:, None]).ravel()
        G = np.stack([np.bincount(key, weights=np.tile(x[:, g], nb), minlength=nb * n_cls) for g in genes], axis=1)
        G = G.reshape(nb, n_cls, genes.size) * np.asarray(inv)[None, :, None]
        for q in range(0, nb, sub):
            Gq = G[q : q + sub]
            shuf = (Gq[:, :, rec][:, a] + Gq[:, :, lig][:, b]).transpose(0, 2, 1)  # [perm][interaction][cluster pair]
            counts += ((shuf > obs) & valid).sum(axis=0)
            ties += int(((shuf == obs) & valid).sum())
    return counts, ties


def observed(x, cl, n_cls):
    sizes = np.bincount(cl, minlength=n_cls).astype(np.float64)
    inv = 1.0 / np.maximum(sizes, 1)
    sums = np.zeros((n_cls, x.shape[1]))
    np.add.at(sums, cl, x)
    return inv, sums * inv[:, None]


def device_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid, **options):
    """``sqb_ligrec_counts`` through a graph-less nhood handle, as ``ligrec_analysis`` drives it, with handle options."""
    lib, ctx = load(), default_context()
    n, n_genes = x.shape
    h = C.c_void_p()
    empty_ptr = np.zeros(n + 1, np.uint32)
    inter32, cp32 = np.ascontiguousarray(inter, np.int32), np.ascontiguousarray(cpairs, np.int32)
    valid_u8 = np.ascontiguousarray(valid, np.uint8)
    data = np.ascontiguousarray(x, np.float64)
    mean_c, inv_c = np.ascontiguousarray(mean_obs, np.float64), np.ascontiguousarray(inv, np.float64)
    counts = np.zeros((inter32.shape[0], cp32.shape[0]), np.int64)
    with ctx.lock:
        check(lib.sqb_nhood_create(ctx.handle, n, 0, empty_ptr.ctypes.data, None, max(n_cls, 2), C.byref(h)))
        try:
            lab = np.ascontiguousarray(cl, np.uint32)
            check(lib.sqb_nhood_set_base(h, lab.ctypes.data, None, 0))
            for k, v in options.items():
                check(lib.sqb_nhood_set_option(h, k.encode(), int(v)))
            st = np.ascontiguousarray(states, np.uint64)
            check(lib.sqb_nhood_permute_upload(h, st.ctypes.data, st.shape[0]))
            check(lib.sqb_ligrec_counts(h, data.ctypes.data, n_genes, inv_c.ctypes.data, mean_c.ctypes.data, inter32.ctypes.data,
                                        inter32.shape[0], cp32.ctypes.data, cp32.shape[0], valid_u8.ctypes.data, counts.ctypes.data))
        finally:
            lib.sqb_nhood_destroy(h)
    return counts


def _all_pairs(n_cls):
    return np.array([(a, b) for a in range(n_cls) for b in range(n_cls)], dtype=np.int64)


def test_fast_reference_equals_oracle():
    x, cl, inter = make_case(0, 300, 10, 5, 30)
    cpairs = _all_pairs(5)
    inv, mean_obs = observed(x, cl, 5)
    states = ref.spawn_states(4, 25)
    valid = np.ones((inter.shape[0], cpairs.shape[0]), bool)
    valid[::3, ::2] = False
    fast, ties = fast_counts(x, cl, 5, states, inv, mean_obs, inter, cpairs, valid, batch=7)
    np.testing.assert_array_equal(fast, ref.ligrec_counts(x, cl, 5, states, inv, mean_obs, inter, cpairs, valid))
    assert ties > 0


@pytest.mark.parametrize("n_cls,near", [(49, False), (120, False), (227, True)])
def test_many_clusters_pvalues_bit_for_bit(n_cls, near):
    optin = smem_optin()
    if near and optin != H100_SMEM_OPTIN:
        pytest.skip(f"C = 227 fills the {H100_SMEM_OPTIN} B opt-in limit of an H100 exactly; this device has {optin} B")
    assert 48 * 1024 < group_means_smem(n_cls) <= optin  # the opt-in launch
    x, cl, inter = make_case(n_cls, 30 * n_cls, 14, n_cls, 24)
    df = pd.DataFrame(x, columns=list(range(x.shape[1])))
    df["clusters"] = pd.Categorical(cl, categories=list(range(n_cls)))
    cpairs = _all_pairs(n_cls)
    P, seed = 40, 9
    res = ligrec_analysis(df, inter, cpairs, threshold=0.0, n_perms=P, seed=seed)
    g = df.groupby("clusters", observed=True)
    mean_obs = g.mean().values
    inv = 1.0 / np.maximum(g.size().values.astype(np.float64), 1)
    valid = ~np.isnan(res.pvalues)
    assert valid.mean() > 0.5
    counts, ties = fast_counts(x, cl, n_cls, spawn_states(seed, P), inv, mean_obs, inter, cpairs, valid)
    np.testing.assert_array_equal(res.pvalues[valid], counts[valid] / P)
    assert ties > 0  # `>` and `>=` differ here


def test_too_many_clusters_is_refused_and_the_context_survives():
    n_cls = 228
    assert group_means_smem(n_cls) > smem_optin()
    x, cl, inter = make_case(1, 20 * n_cls, 6, n_cls, 8)
    df = pd.DataFrame(x, columns=list(range(x.shape[1])))
    df["clusters"] = pd.Categorical(cl, categories=list(range(n_cls)))
    with pytest.raises(NotImplementedError, match="228 clusters exceed the shared-memory accumulators"):
        ligrec_analysis(df, inter, _all_pairs(n_cls), threshold=0.0, n_perms=10, seed=1)
    x, cl, inter = make_case(2, 400, 8, 6, 16)
    cpairs = _all_pairs(6)
    inv, mean_obs = observed(x, cl, 6)
    states = spawn_states(3, 20)
    valid = np.ones((inter.shape[0], cpairs.shape[0]), bool)
    got = device_counts(x, cl, 6, states, inv, mean_obs, inter, cpairs, valid)
    np.testing.assert_array_equal(got, fast_counts(x, cl, 6, states, inv, mean_obs, inter, cpairs, valid)[0])


def test_four_chunks_through_perm_chunk():
    n_cls, P = 8, 100
    x, cl, inter = make_case(5, 600, 12, n_cls, 30)
    cpairs = _all_pairs(n_cls)
    assert perm_chunks(P, upload_chunk(P, perm_chunk=32), n_cls, x.shape[1]) == [32, 32, 32, 4]
    inv, mean_obs = observed(x, cl, n_cls)
    states = spawn_states(6, P)
    valid = np.ones((inter.shape[0], cpairs.shape[0]), bool)
    valid[1::4] = False
    exp, ties = fast_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid)
    assert ties > 0
    np.testing.assert_array_equal(device_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid, perm_chunk=32), exp)
    np.testing.assert_array_equal(device_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid), exp)  # one chunk


def test_group_means_cap_splits_the_default_chunk():
    """n = 500, C = 60, G = 200, P = 12 000: the [perm][cluster][gene] means are capped at 1 GB, 11 184 permutations per
    pass, so the default upload chunk (12 000) runs as 11 184 + 816.  Only a few genes take part in interactions, which
    keeps the reference cheap; the device forms the means of all 200."""
    n_cls, n_genes, P, n = 60, 200, 12000, 500
    assert upload_chunk(P, stride=n) == 12000
    assert perm_chunks(P, upload_chunk(P, stride=n), n_cls, n_genes) == [11184, 816]
    rng = np.random.default_rng(7)
    x = rng.poisson(0.8, size=(n, n_genes)).astype(np.float64)
    cl = rng.integers(0, n_cls, n)
    cl[:n_cls] = np.arange(n_cls)
    genes = rng.choice(n_genes, 6, replace=False)
    inter = np.array([(genes[i], genes[j]) for i in range(6) for j in range(6) if i != j][:12])
    cpairs = _all_pairs(n_cls)
    inv, mean_obs = observed(x, cl, n_cls)
    states = spawn_states(8, P)
    valid = np.ones((inter.shape[0], cpairs.shape[0]), bool)
    exp, ties = fast_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid, batch=2000)
    assert ties > 0
    got = device_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid)
    np.testing.assert_array_equal(got, exp)
    assert (got > 816).any()  # counts from both passes: the first alone cannot exceed 11 184, the second alone not 816


@pytest.mark.parametrize("n,algo", [(70000, 7), (524288, 9)])
def test_labels_from_the_list_and_region_replays(n, algo):
    n_cls, P = 7, 300
    sm = default_context().sm_count
    x, cl, inter = make_case(n, n, 3, n_cls, 6, lam=0.3)
    chunks = perm_chunks(P, upload_chunk(P, stride=n), n_cls, x.shape[1])
    assert chunks == [P] and auto_replay(n, P, sm) == algo
    cpairs = _all_pairs(n_cls)
    inv, mean_obs = observed(x, cl, n_cls)
    states = spawn_states(n + 1, P)
    valid = np.ones((inter.shape[0], cpairs.shape[0]), bool)
    exp, _ = fast_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid, batch=32)
    np.testing.assert_array_equal(device_counts(x, cl, n_cls, states, inv, mean_obs, inter, cpairs, valid), exp)
    assert 0 < exp.sum() < P * exp.size
