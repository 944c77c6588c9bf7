"""``nhood_enrichment`` — drop-in for ``squidpy.gr.nhood_enrichment`` (``src/squidpy/gr/_nhood.py:146-242``) running the
permutation test on an H100 through ``libsquidpy_b200.so``; ``interaction_matrix`` and ``centrality_scores`` over the same
neighbour graph.

Same signature, same ``adata.uns`` keys, same exceptions.  ``numba_parallel``, ``n_jobs``, ``backend`` and
``show_progress_bar`` are accepted for compatibility and ignored (the joblib fan-out over permutations is replaced by
one CTA per permutation on the GPU).  Extra keyword-only argument: ``device``.
Z-scores are computed on the host from the per-permutation uint32 counts exactly like the reference
(float64 ``mean``/``std`` over permutations, :231), so with the same ``seed`` they are identical to the reference's.
"""

from __future__ import annotations

import ctypes as C
import threading
import time
from typing import Any, NamedTuple

import numpy as np

from .._constants import Centrality, Key
from .._device import DevGraph, device_graph, graph_args, graph_value_code
from .._dist import nccl_cuda, sequential_stats, shard_range, shared_seed, stats_device, world
from .._lib import Context, check, default_context, load
from .._rng import spawn_states
from .._validators import assert_categorical_obs, assert_connectivity_key, assert_positive, extract_adata_if_sdata
from ._utils import _save_data, as_csr, caller_graph, category_codes, logg
from ._utils import graph_device as _graph_device

__all__ = ["nhood_enrichment", "NhoodEnrichmentResult", "NhoodPlan", "centrality_scores", "centrality_counts"]


class NhoodEnrichmentResult(NamedTuple):
    """Result of :func:`nhood_enrichment` (``_nhood.py:44-48``)."""

    zscore: np.ndarray
    counts: np.ndarray  # 'count' clashes with tuple.count


def _as_u32(a) -> np.ndarray:
    """uint32 view of a CSR index array (reference: ``.astype(uint32)``, ``_nhood.py:205``).  int32 input is
    re-interpreted in place — no copy, so page-locked caller buffers stay page-locked for the H2D copy."""
    a = np.asarray(a)
    if a.dtype == np.int32 and a.flags.c_contiguous:
        return a.view(np.uint32)  # a negative index becomes >= 2^31 and is rejected by the device-side range check
    if a.dtype.kind == "i" and a.size and a.min() < 0:
        raise ValueError("Negative CSR index.")
    return np.ascontiguousarray(a, dtype=np.uint32)


class NhoodPlan:
    """Device-resident neighbour graph (CSR) + kernels: the object behind the C-ABI handle ``sqb_nhood``.

    ``count(labels)`` replaces ``_test(indices, indptr, clustering)`` (``_nhood.py:208-209``);
    ``permute(states)`` replaces ``_nhood_enrichment_helper`` over all permutations (``_nhood.py:516-547``)."""

    def __init__(self, indptr: np.ndarray, indices: np.ndarray, n_cls: int, ctx: Context | None = None):
        self._lib = load()
        self.ctx = ctx or default_context()
        self.indptr = _as_u32(indptr)
        self.indices = _as_u32(indices)
        self.n = self.indptr.size - 1
        self.n_cls = int(n_cls)
        h = C.c_void_p()
        check(
            self._lib.sqb_nhood_create(self.ctx.handle, self.n, self.indices.size, self.indptr.ctypes.data,
                                       self.indices.ctypes.data, self.n_cls, C.byref(h))
        )
        self._h = h
        self.n_perms = 0

    @classmethod
    def from_device(cls, graph: DevGraph, n_cls: int, ctx: Context | None = None) -> "NhoodPlan":
        """Plan over a neighbour graph already in GPU memory (``graph_args`` of a cupy-style or torch CSR / CSC).  The library
        converts and validates it into its own copy on the device and never reads it on the host.  The caller may free the
        graph when this returns.  For a CSC graph the plan holds the transpose: its counts are the transposes of the
        graph's (``graph.transposed``)."""
        self = cls.__new__(cls)
        self._h = None
        self._lib = load()
        self.ctx = ctx or default_context()
        self.indptr = self.indices = None  # no host copy
        self.n = graph.n
        self.n_cls = int(n_cls)
        h = C.c_void_p()
        check(
            self._lib.sqb_nhood_create_device(self.ctx.handle, graph.n, graph.nnz, graph.indptr, graph.indptr_bits, graph.indices or None,
                                              graph.index_bits, self.n_cls, graph.stream, C.byref(h))
        )
        self._h = h
        self.n_perms = 0
        return self

    def set_option(self, key: str, value: int) -> None:
        check(self._lib.sqb_nhood_set_option(self._h, key.encode(), int(value)))

    @property
    def bytes_per_perm(self) -> int:
        b = C.c_int64()
        check(self._lib.sqb_nhood_bytes_per_perm(self._h, C.byref(b)))
        return b.value

    def count(self, labels: np.ndarray) -> np.ndarray:
        labels = np.ascontiguousarray(labels, dtype=np.uint32)
        if labels.size != self.n:
            raise ValueError(f"Expected `{self.n}` labels, found `{labels.size}`.")
        out = np.empty((self.n_cls, self.n_cls), dtype=np.uint32)
        check(self._lib.sqb_nhood_count(self._h, labels.ctypes.data, out.ctypes.data))
        return out

    def set_base(self, labels: np.ndarray, lib_codes: np.ndarray | None = None, n_libs: int = 0) -> None:
        labels = np.ascontiguousarray(labels, dtype=np.uint32)
        if labels.size != self.n:
            raise ValueError(f"Expected `{self.n}` labels, found `{labels.size}`.")
        lc = None if lib_codes is None else np.ascontiguousarray(lib_codes, dtype=np.int32)
        check(self._lib.sqb_nhood_set_base(self._h, labels.ctypes.data, None if lc is None else lc.ctypes.data, int(n_libs)))

    def upload(self, states: np.ndarray) -> None:
        states = np.ascontiguousarray(states, dtype=np.uint64)
        if states.ndim != 2 or states.shape[1] != 6:
            raise ValueError("Expected generator states of shape (n_perms, 6).")
        check(self._lib.sqb_nhood_permute_upload(self._h, states.ctypes.data, states.shape[0]))
        self.n_perms = states.shape[0]

    def upload_philox(self, seed: int, first_perm: int, n_perms: int) -> None:
        """Fast RNG mode: permutations ``first_perm .. first_perm + n_perms`` of the keyed-bijection family ``seed`` (see
        ``sqb_nhood_permute_upload_philox``); nothing but three integers is uploaded."""
        check(self._lib.sqb_nhood_permute_upload_philox(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF, int(first_perm), int(n_perms)))
        self.n_perms = int(n_perms)

    def run_async(self) -> None:
        check(self._lib.sqb_nhood_permute_run_async(self._h))

    def download(self, out: np.ndarray | None = None) -> np.ndarray:
        if out is None:
            out = np.empty((self.n_perms, self.n_cls, self.n_cls), dtype=np.uint32)
        check(self._lib.sqb_nhood_permute_download(self._h, out.ctypes.data))
        return out

    def stats(self) -> tuple[np.ndarray, np.ndarray]:
        """float64 (n_cls, n_cls) mean and standard deviation over the permutations of the last run, bit-identical to
        ``perms.astype(float64).mean(axis=0)`` / ``.std(axis=0)`` (same operation order, computed on the device)."""
        mean = np.empty((self.n_cls, self.n_cls), dtype=np.float64)
        std = np.empty((self.n_cls, self.n_cls), dtype=np.float64)
        check(self._lib.sqb_nhood_permute_stats(self._h, mean.ctypes.data, std.ctypes.data))
        return mean, std

    def sums(self) -> np.ndarray:
        """int64 (n_cls, n_cls) exact per-bin sums over this plan's permutations (multi-GPU statistics, see ``_dist``)."""
        out = np.empty((self.n_cls, self.n_cls), dtype=np.int64)
        check(self._lib.sqb_nhood_permute_sums(self._h, out.ctypes.data))
        return out

    def var_chain(self, mean: np.ndarray, acc_in: np.ndarray) -> np.ndarray:
        """Continue numpy's sequential ``sum((x - mean)**2)`` over this plan's permutations from ``acc_in``."""
        mean = np.ascontiguousarray(mean, dtype=np.float64)
        acc_in = np.ascontiguousarray(acc_in, dtype=np.float64)
        out = np.empty((self.n_cls, self.n_cls), dtype=np.float64)
        check(self._lib.sqb_nhood_permute_var_chain(self._h, mean.ctypes.data, acc_in.ctypes.data, out.ctypes.data))
        return out

    def stats_dev(self, d_mean: int, d_std: int) -> None:
        """``stats`` into caller-owned device buffers (raw pointers), asynchronous on the context's stream."""
        check(self._lib.sqb_nhood_permute_stats_dev(self._h, C.c_void_p(d_mean), C.c_void_p(d_std)))

    def sums_dev(self, d_sums: int) -> None:
        check(self._lib.sqb_nhood_permute_sums_dev(self._h, C.c_void_p(d_sums)))

    def counts_dev(self, d_dst: int) -> None:
        """Asynchronous device-to-device copy of the per-permutation counts [n_perms, C*C] (uint32) to ``d_dst``."""
        check(self._lib.sqb_nhood_permute_counts_dev(self._h, C.c_void_p(d_dst)))

    def var_chain_dev(self, d_mean: int, d_acc_in: int, d_acc_out: int) -> None:
        check(self._lib.sqb_nhood_permute_var_chain_dev(self._h, C.c_void_p(d_mean), C.c_void_p(d_acc_in), C.c_void_p(d_acc_out)))

    def permute(self, states: np.ndarray) -> np.ndarray:
        """uint32 (n_perms, n_cls, n_cls) neighbour-pair counts of every permutation."""
        states = np.ascontiguousarray(states, dtype=np.uint64)
        out = np.empty((states.shape[0], self.n_cls, self.n_cls), dtype=np.uint32)
        check(self._lib.sqb_nhood_permute(self._h, states.ctypes.data, states.shape[0], out.ctypes.data))
        self.n_perms = states.shape[0]
        return out

    def shuffled_labels(self, p0: int, p1: int) -> np.ndarray:
        out = np.empty((p1 - p0, self.n), dtype=np.uint32)
        check(self._lib.sqb_nhood_shuffled_labels(self._h, p0, p1, out.ctypes.data))
        return out

    def close(self) -> None:
        if self._h is not None:
            self._lib.sqb_nhood_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


def nhood_enrichment(
    adata: Any,
    cluster_key: str,
    library_key: str | None = None,
    connectivity_key: str | None = None,
    n_perms: int = 1000,
    numba_parallel: bool = False,
    seed: int | None = None,
    copy: bool = False,
    n_jobs: int | None = None,
    backend: str = "loky",
    show_progress_bar: bool = True,
    *,
    table_key: str | None = None,
    device: int | None = None,
    rng: str = "numpy",
) -> NhoodEnrichmentResult | None:
    """Compute neighborhood enrichment by permutation test (see module docstring).

    ``rng="numpy"`` (default) replays the reference's permutations bit-exactly (``spawn_generators`` + ``Generator.shuffle``):
    z-scores identical to the reference for the same ``seed``.  ``rng="philox"`` draws the permutations from a keyed
    bijection evaluated on the device instead (same null distribution, different draws, ~4x faster): z-scores agree with
    the exact mode to O(n_perms^-1/2), not bit-wise.

    Returns ``NhoodEnrichmentResult(zscore, counts)`` if ``copy=True``; otherwise writes
    ``adata.uns[f'{cluster_key}_nhood_enrichment'] = {'zscore': float64[C,C], 'count': uint32[C,C]}``.
    Under an initialised ``torch.distributed`` process group (one process per GPU) the permutations are sharded
    over the ranks and the per-permutation counts all-gathered once; every rank gets the full result."""
    adata = extract_adata_if_sdata(adata, table_key=table_key)
    connectivity_key = Key.obsp.spatial_conn(connectivity_key)
    assert_categorical_obs(adata, cluster_key)
    assert_connectivity_key(adata, connectivity_key)
    assert_positive(n_perms, name="n_perms")

    # a graph in GPU memory is read there (converted into the plan's own copy); a host graph goes through scipy as before
    dev = device_graph(adata.obsp[connectivity_key])
    graph = None if dev is None else graph_args(dev, adata.shape[0])
    if dev is None:
        adj = as_csr(adata.obsp[connectivity_key])
    int_clust, n_cls = category_codes(adata.obs[cluster_key], dtype=np.uint32)
    if n_cls <= 1:
        raise ValueError(f"Expected at least `2` clusters, found `{n_cls}`.")  # _nhood.py:107-108

    lib_codes, n_libs = None, 0
    if library_key is not None:
        assert_categorical_obs(adata, key=library_key)
        libs = adata.obs[library_key]
        lib_codes = np.asarray(libs.array.codes).astype(np.int32)
        n_libs = len(libs.cat.categories)

    if rng not in ("numpy", "philox"):
        raise ValueError(f"Expected `rng` to be 'numpy' or 'philox', found `{rng!r}`.")
    start = time.perf_counter()
    if graph is not None:
        device = _graph_device(dev, device)
    ctx = default_context(device)
    rank, ws = world()
    lo, hi = shard_range(int(n_perms), rank, ws)
    seed = shared_seed(seed)  # seed=None: one entropy draw for all ranks (every rank must spawn the same family)
    # the PCG64 states of this rank's generators are spawned on a host thread while the graph goes to the device
    # (the C calls below release the GIL)
    states_box: list = []
    spawner = None
    if hi > lo and rng == "numpy":
        spawner = threading.Thread(target=lambda: states_box.append(spawn_states(seed, int(n_perms), lo, hi)), daemon=True)
        spawner.start()
    with ctx.lock:
        plan = NhoodPlan(adj.indptr, adj.indices, n_cls, ctx) if graph is None else NhoodPlan.from_device(graph, n_cls, ctx)
        try:
            count = plan.count(int_clust)
            logg.info("Calculating neighborhood enrichment on cuda:%d (rank %d/%d, permutations %d..%d)", ctx.device, rank, ws, lo, hi)
            if hi > lo:
                plan.set_base(int_clust, lib_codes, n_libs)
                if rng == "philox":
                    plan.upload_philox(int(np.random.SeedSequence(seed).generate_state(1, np.uint64)[0]), lo, hi - lo)
                else:
                    spawner.join()
                    if not states_box:  # the spawn raised (e.g. too many children): repeat it here for the exception
                        states_box.append(spawn_states(seed, int(n_perms), lo, hi))
                    plan.upload(states_box[0])
                plan.run_async()
            if ws == 1:
                # single GPU: mean / std over the permutations on the device, in numpy's operation order (bit-identical to
                # the host expression of the reference); the per-permutation counts never leave the GPU
                mean, std = plan.stats()
            elif nccl_cuda():
                # several GPUs: the per-permutation counts of all ranks are all-gathered as device tensors (one collective) and
                # every rank runs the same statistics kernel over them; one [2, C, C] download.  (Very large count arrays: exact
                # integer sums all-reduced + the order-dependent variance accumulation chained through the ranks.)  Either way
                # bit-identical to mean/std of the gathered counts.
                mean, std = stats_device(plan, int(n_perms), hi > lo)
            else:  # gloo (CPU tests of the host logic): the same chain through host buffers
                if hi > lo:
                    sums_local, step = plan.sums(), plan.var_chain
                else:  # more ranks than permutations
                    sums_local, step = np.zeros((n_cls, n_cls), dtype=np.int64), (lambda mean, acc: acc)
                mean, std = sequential_stats(sums_local, step, int(n_perms))
        finally:
            plan.close()
    if graph is not None and graph.transposed:
        # the plan held the CSC graph's transpose: every per-permutation count is transposed, hence count, mean and std
        # bin for bin
        count, mean, std = (np.ascontiguousarray(a.T) for a in (count, mean, std))
    with np.errstate(divide="ignore", invalid="ignore"):
        zscore = (count - mean) / std  # _nhood.py:231 (no zero-std guard there either)

    if copy:
        return NhoodEnrichmentResult(zscore=zscore, counts=count)
    _save_data(adata, attr="uns", key=Key.uns.nhood_enrichment(cluster_key), data={"zscore": zscore, "count": count},
               time_start=start)
    return None


class CentralityCounts(NamedTuple):
    """The integer parts of the group measures (``sqb_centrality_scores``); fields not requested are ``None``."""

    reach1: np.ndarray | None  # int64[C]: |N(S) \ S|
    dist: np.ndarray | None  # int64[C]: sum of hop distances from S over the nodes it reaches
    cc: np.ndarray | None  # float64[n]: local clustering coefficient
    levels: int  # BFS levels that reached a node (-1 without closeness)


# value dtype of a host graph -> (dtype it is uploaded as, ABI value code, bits at which its integer sum wraps)
_HOST_VALUES = {
    np.dtype(np.bool_): (np.bool_, 5, 64), np.dtype(np.float32): (np.float32, 0, 64), np.dtype(np.float64): (np.float64, 1, 64),
    np.dtype(np.int8): (np.int32, 3, 8), np.dtype(np.uint8): (np.int32, 3, 8), np.dtype(np.int16): (np.int32, 3, 16),
    np.dtype(np.uint16): (np.int32, 3, 16), np.dtype(np.int32): (np.int32, 3, 32), np.dtype(np.uint32): (np.int64, 4, 32),
    np.dtype(np.int64): (np.int64, 4, 64), np.dtype(np.uint64): (np.int64, 4, 64),
}
_MEASURE_BITS = {Centrality.DEGREE: 1, Centrality.CLOSENESS: 2, Centrality.CLUSTERING: 4}


def centrality_counts(conn: Any, codes: np.ndarray, n_cls: int, measures: int, *, device: int | None = None) -> CentralityCounts:
    """Run ``sqb_centrality_scores`` on the neighbour graph ``conn``: a scipy / numpy matrix on the host, or a CSR / CSC
    in GPU memory (as ``nhood_enrichment`` takes it).  ``codes``: int32[n] cluster codes, -1 for none.  ``measures``: a
    mask of 1 (degree), 2 (closeness), 4 (clustering).  A CSC matrix is read as the CSR of its transpose, which is the
    same undirected graph."""
    codes = np.ascontiguousarray(codes, dtype=np.int32)
    n = codes.size
    g = caller_graph(conn, n, device)
    if g.dev is None:
        spec = _HOST_VALUES.get(g.host.dtype)
        if spec is None:
            raise TypeError(f"Graph values of dtype `{g.host.dtype}` are not supported.")
        dtype, code, int_bits = spec
        data = g.host.data.view(np.int64) if g.host.dtype == np.uint64 else g.host.data
        data = np.ascontiguousarray(data, dtype=dtype)
        data_ptr = data.ctypes.data
    else:
        code = graph_value_code(g.dev.data, g.index_args[1])
        if code == 2:
            raise TypeError("Device graph values of dtype `float16` are not supported; use float32, float64, int32, int64 or bool.")
        int_bits, data_ptr = 32 if code == 3 else 64, g.dev.data.ptr or None
    args = (*g.index_args, data_ptr, code, int_bits, int(g.dev is not None))
    reach1 = np.zeros(n_cls, dtype=np.int64) if measures & 1 else None
    dist = np.zeros(n_cls, dtype=np.int64) if measures & 2 else None
    cc = np.empty(n, dtype=np.float64) if measures & 4 else None
    levels = C.c_int64(-1)
    ctx = default_context(g.device)
    with ctx.lock:
        check(load().sqb_centrality_scores(ctx.handle, *args, codes.ctypes.data, int(n_cls), int(measures),
                                           None if reach1 is None else reach1.ctypes.data, None if dist is None else dist.ctypes.data,
                                           None if cc is None else cc.ctypes.data, C.byref(levels), g.stream))
    return CentralityCounts(reach1, dist, cc, int(levels.value))


def centrality_scores(
    adata: Any,
    cluster_key: str,
    score: str | Centrality | None = None,
    connectivity_key: str | None = None,
    copy: bool = False,
    n_jobs: int | None = None,
    backend: str = "loky",
    show_progress_bar: bool = False,
    *,
    table_key: str | None = None,
    device: int | None = None,
):
    """Centrality scores of every cluster (reference ``gr/_nhood.py:245-346``) over the undirected neighbour graph
    ``obsp[connectivity_key] + obsp[connectivity_key].T`` without self loops, entries whose sum is zero dropped.  For the
    group S of each category (``cat.categories`` in order, unused ones included; observations with a NaN label are nodes of
    the graph but in no group) and n observations:

    - ``degree_centrality``: ``|N(S) \\ S| / (n - |S|)``;
    - ``average_clustering``: the mean over S of the local clustering coefficient, 0.0 for an empty group;
    - ``closeness_centrality``: ``(n - |S|) / sum of d(S, v)`` over the nodes v outside S reachable from S in hops, 0.0
      when that sum is 0.

    Where the measure is undefined the value is NaN: closeness of an empty category and degree of a category holding every
    observation.  The counts are computed on the GPU (``centrality_counts``), the divisions on the host in float64, so the
    values are those of networkx's ``group_degree_centrality`` / ``group_closeness_centrality`` / ``average_clustering``.

    ``score``: one name (``str`` or :class:`Centrality`) or ``None`` for all three, in that order: degree, clustering,
    closeness.  ``n_jobs``, ``backend`` and ``show_progress_bar`` are accepted and ignored.  Under a process group every
    rank computes the whole result on its own device.  Returns the float64 frame if ``copy=True``, otherwise writes
    ``adata.uns[f'{cluster_key}_centrality_scores']``."""
    import pandas as pd

    adata = extract_adata_if_sdata(adata, table_key=table_key)
    connectivity_key = Key.obsp.spatial_conn(connectivity_key)
    assert_categorical_obs(adata, cluster_key)
    assert_connectivity_key(adata, connectivity_key)
    if isinstance(score, str | Centrality):
        centrality = [score]
    elif score is None:
        centrality = [c.s for c in Centrality]
    else:  # the reference leaves `centrality` unbound here (:293-298)
        raise UnboundLocalError("cannot access local variable 'centrality' where it is not associated with a value")
    centralities = [Centrality(c) for c in centrality]

    start = time.perf_counter()
    cats = adata.obs[cluster_key]
    cat = cats.cat.categories.values
    n_cls = len(cat)
    codes = np.asarray(cats.array.codes, dtype=np.int32)
    n = codes.size
    measures = 0
    for c in centralities:
        measures |= _MEASURE_BITS[c]
    counts = centrality_counts(adata.obsp[connectivity_key], codes, n_cls, measures, device=device)
    logg.info("Calculating centralities `%s` on the GPU (%d BFS levels)", centralities, counts.levels)

    size = np.bincount(codes[codes >= 0], minlength=n_cls)
    columns = {}
    for c in centralities:
        if c == Centrality.DEGREE:  # networkx: len(N(S) - S) / (len(G) - len(S)), Python int division
            vals = [int(r) / (n - int(s)) if n != s else np.nan for r, s in zip(counts.reach1, size)]
        elif c == Centrality.CLOSENESS:
            vals = [np.nan if s == 0 else ((n - int(s)) / int(d) if d else 0.0) for d, s in zip(counts.dist, size)]
        else:  # float(cc[idx].mean()) per group (:316): the group's coefficients in index order, numpy's pairwise mean
            order = np.argsort(codes, kind="stable")[n - int(size.sum()):]
            groups = np.split(counts.cc[order], np.cumsum(size)[:-1])
            vals = [float(g.mean()) if g.size else 0.0 for g in groups]
        columns[c.s] = pd.DataFrame(vals, columns=[c.s], index=cat)
    df = pd.concat(list(columns.values()), axis=1)

    if copy:
        return df
    _save_data(adata, attr="uns", key=Key.uns.centrality_scores(cluster_key), data=df, time_start=start)
    return None


def interaction_matrix(
    adata: Any,
    cluster_key: str,
    connectivity_key: str | None = None,
    normalized: bool = False,
    copy: bool = False,
    weights: bool = False,
    *,
    table_key: str | None = None,
    device: int | None = None,
) -> np.ndarray | None:
    """Compute the interaction matrix of the clusters (reference ``gr/_nhood.py:349-409``): entry (a, b) sums the stored
    entries (i -> j) of ``obsp[connectivity_key]`` with cluster(i) = a and cluster(j) = b, their values if ``weights`` else
    ones; observations with a NaN label are dropped from rows and columns; ``normalized`` divides every row by its sum.
    dtype as in the reference (:398): int64 for bool / integer graphs, float64 otherwise.

    Returns the matrix if ``copy=True``, otherwise writes ``adata.uns[f'{cluster_key}_interactions']``."""
    import pandas as pd

    adata = extract_adata_if_sdata(adata, table_key=table_key)
    connectivity_key = Key.obsp.spatial_conn(connectivity_key)
    assert_categorical_obs(adata, cluster_key)
    assert_connectivity_key(adata, connectivity_key)

    cats = adata.obs[cluster_key]
    codes = np.ascontiguousarray(cats.array.codes, dtype=np.int32)  # -1 == NaN label
    if not (codes >= 0).any():
        raise RuntimeError(f"After removing NaNs in `adata.obs[{cluster_key!r}]`, none remain.")  # _nhood.py:391-392
    dev = device_graph(adata.obsp[connectivity_key])
    if dev is None:
        g = as_csr(adata.obsp[connectivity_key])
        value_dtype = g.dtype
    else:  # read in place on the device
        graph = graph_args(dev, adata.shape[0])
        value_dtype = dev.data.dtype
        device = _graph_device(dev, device)
    n_cats = len(cats.cat.categories)
    int_graph = bool(pd.api.types.is_bool_dtype(value_dtype) or pd.api.types.is_integer_dtype(value_dtype))

    ctx = default_context(device)
    lib = load()
    if weights:
        out = np.zeros((n_cats, n_cats), dtype=np.float64)
        if dev is not None:
            _interaction_device(lib, ctx, graph, codes, n_cats, out, None)
        else:
            indptr, indices = _as_u32(g.indptr), _as_u32(g.indices)
            data = g.data
            if data.dtype not in (np.float32, np.float64):
                data = data.astype(np.float64)  # integer / bool weights are summed exactly in float64 (< 2^53)
            data = np.ascontiguousarray(data)
            check(lib.sqb_interaction_matrix(ctx.handle, g.shape[0], indices.size, indptr.ctypes.data, indices.ctypes.data,
                                             data.ctypes.data, 0 if data.dtype == np.float32 else 1, codes.ctypes.data, n_cats,
                                             out.ctypes.data, None))
        output = np.rint(out).astype(np.int64) if int_graph else out
    else:
        cnt = np.zeros((n_cats, n_cats), dtype=np.int64)
        if dev is not None:
            _interaction_device(lib, ctx, graph, codes, n_cats, None, cnt)
        else:
            indptr, indices = _as_u32(g.indptr), _as_u32(g.indices)
            check(lib.sqb_interaction_matrix(ctx.handle, g.shape[0], indices.size, indptr.ctypes.data, indices.ctypes.data,
                                             None, 0, codes.ctypes.data, n_cats, None, cnt.ctypes.data))
        output = cnt if int_graph else cnt.astype(np.float64)
    if normalized:
        with np.errstate(divide="ignore", invalid="ignore"):
            output = output / output.sum(axis=1).reshape((-1, 1))  # _nhood.py:403-404
    if copy:
        return output
    _save_data(adata, attr="uns", key=Key.uns.interaction_matrix(cluster_key), data=output)
    return None


def _interaction_device(lib, ctx: Context, graph: DevGraph, codes: np.ndarray, n_cats: int, out_w: np.ndarray | None,
                        out_c: np.ndarray | None) -> None:
    """Sums (``out_w``, float64) or counts (``out_c``, int64) of a device graph into the host matrix given, read in place by
    ``sqb_interaction_matrix_device``; transposed back for a CSC graph."""
    vals = graph.sparse.data
    code = graph_value_code(vals, graph.nnz) if out_w is not None else 0
    out = out_w if out_w is not None else out_c
    with ctx.lock:
        check(lib.sqb_interaction_matrix_device(ctx.handle, graph.n, graph.nnz, graph.indptr, graph.indptr_bits, graph.indices or None,
                                                graph.index_bits, (vals.ptr or None) if out_w is not None else None, code,
                                                codes.ctypes.data, n_cats, None if out_w is None else out_w.ctypes.data,
                                                None if out_c is None else out_c.ctypes.data, graph.stream))
    if graph.transposed:
        out[...] = out.T.copy()
