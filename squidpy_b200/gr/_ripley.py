"""``ripley`` — drop-in for ``squidpy.gr.ripley`` (``src/squidpy/gr/_ripley.py:27-194``).

Mode ``L``: the expensive step — cumulative ordered-pair counts per cluster, ``KDTree.two_point_correlation`` in the
reference (:218-223) — runs on the H100 (``sqb_pair_counts_f64``: float64, bit-identical counts), for the observed
clusters and for all Poisson-point-process simulations in ONE launch.  This holds for all nine metric names ``KDTree``
takes: each resolves to scikit-learn's euclidean, manhattan or chebyshev distance, and the kernel computes all three in
float64 exactly as scikit-learn does.  Modes ``F``/``G``: the nearest-neighbour searches (:140-150, :160-169) and the
histogram of their distances (:206-209) run on the H100 too (``sqb_nn_dist_hist_f64``: float64,
bit-identical bin counts) for the euclidean metric, again in ONE call for the observed clusters and every simulation.  G is
the heavy one: its observed statistic queries every point outside a cluster against the cluster, and every simulation
queries all N points.  A reference set goes to the device only when scikit-learn would search it with its kd_tree (whose
distances the kernel reproduces bit for bit); smaller sets, where scikit-learn switches to brute force and its GEMM-form
distances, and every other metric stay on the host with scikit-learn.  The convex hull, the rejection-sampled simulations
(they must consume numpy's RNG stream exactly), the cumulative fractions and the long-format reshaping stay on the host.
"""

from __future__ import annotations

import time
from typing import Any, Literal

import numpy as np
import pandas as pd

from .._constants import Key, RipleyStat
from .._device import on_host
from .._dist import all_reduce_sum, world, shared_seed
from .._lib import Context, check, default_context, load
from .._metrics import metric_code
from .._rng import spawn_generators
from .._validators import assert_categorical_obs, assert_spatial_basis, extract_adata_if_sdata
from ._utils import _save_data, logg

__all__ = ["ripley", "pair_counts", "nn_distance_hist"]

# metrics NearestNeighbors searches with the euclidean distance (minkowski: its default p = 2)
_EUCLIDEAN = ("euclidean", "l2", "minkowski")
_NN_MAX_K = 64  # largest k of the kernel


def pair_counts(groups: list[np.ndarray], support: np.ndarray, *, metric: int = 0, ctx: Context | None = None,
                shard: tuple[int, int] = (0, 1)) -> np.ndarray:
    """For every point set in ``groups`` (each (m, 2) float64): int64 (len(groups), S) counts of ordered pairs, self pairs
    included, with ``d(p, q) <= support[s]`` — i.e. ``KDTree(p, metric=m).two_point_correlation(p, support)``.  ``metric``
    (see :func:`squidpy_b200._metrics.metric_code`): 0 euclidean ``sqrt(dx^2 + dy^2)``, 1 manhattan ``|dx| + |dy|``, 2 chebyshev
    ``max(|dx|, |dy|)``.  ``shard=(r, n)``: this device's share of the pair tiles (the shares add up to the whole)."""
    lib = load()
    ctx = ctx or default_context()
    support = np.ascontiguousarray(support, dtype=np.float64)
    ptr = np.zeros(len(groups) + 1, dtype=np.int64)
    ptr[1:] = np.cumsum([len(g) for g in groups])
    pts = np.ascontiguousarray(np.concatenate([np.asarray(g, dtype=np.float64).reshape(-1, 2) for g in groups], axis=0)) if ptr[-1] else np.zeros((1, 2))
    out = np.empty((len(groups), support.size), dtype=np.int64)
    check(lib.sqb_pair_counts_f64(ctx.handle, pts.ctypes.data, ptr.ctypes.data, len(groups), support.ctypes.data, support.size,
                                  int(metric), int(shard[0]), int(shard[1]), out.ctypes.data))
    return out


def nn_distance_hist(points: np.ndarray, tasks: np.ndarray, support: np.ndarray, n_rows: int, *, ctx: Context | None = None,
                     shard: tuple[int, int] = (0, 1)) -> np.ndarray:
    """Histograms of nearest-neighbour distances on the GPU: int64 (n_rows, len(support) - 1).

    ``points`` is an (n, 2) pool of float64 coordinates; every row of ``tasks`` (int64, 6 columns) is ``(ref_begin, ref_end,
    qry_begin, qry_end, k, row)``: the k nearest distances of every query point ``points[qry_begin:qry_end]`` among
    ``points[ref_begin:ref_end]`` (no point excluded) are added to histogram ``row``, i.e.
    ``np.histogram(NearestNeighbors().fit(ref).kneighbors(qry, k)[0], bins=support)[0]`` with scikit-learn's kd_tree
    distances.  ``support`` must be ascending; 1 <= k <= min(64, ref_end - ref_begin).  ``shard=(r, n)``: this device's share of
    the query blocks (the shares add up to the whole)."""
    lib = load()
    ctx = ctx or default_context()
    pts = np.ascontiguousarray(np.asarray(points, dtype=np.float64).reshape(-1, 2))
    tk = np.ascontiguousarray(np.asarray(tasks, dtype=np.int64).reshape(-1, 6))
    support = np.ascontiguousarray(support, dtype=np.float64)
    out = np.empty((int(n_rows), max(support.size - 1, 0)), dtype=np.int64)
    check(lib.sqb_nn_dist_hist_f64(ctx.handle, pts.ctypes.data if pts.size else np.zeros(2).ctypes.data, pts.shape[0], tk.ctypes.data, tk.shape[0],
                                   support.ctypes.data, support.size, int(n_rows), int(shard[0]), int(shard[1]), out.ctypes.data))
    return out


def ripley(
    adata: Any,
    cluster_key: str,
    mode: Literal["F", "G", "L"] = "F",
    spatial_key: str = Key.obsm.spatial,
    metric: str = "euclidean",
    n_neigh: int = 2,
    n_simulations: int = 100,
    n_observations: int = 1000,
    max_dist: float | None = None,
    n_steps: int = 50,
    seed: int | None = None,
    copy: bool = False,
    *,
    table_key: str | None = None,
    device: int | None = None,
) -> dict[str, pd.DataFrame | np.ndarray] | None:
    """Calculate Ripley's F, G or L statistics (see module docstring).

    Result dict (``copy=True``) or ``adata.uns[f'{cluster_key}_ripley_{mode}']``: ``{f'{mode}_stat'``: long DataFrame
    (bins, cluster, stats), ``'sims_stat'``: long DataFrame, ``'bins'``: float64[n_steps], ``'pvalues'``:
    float64[n_clusters, n_steps]``}``."""
    from scipy.spatial import ConvexHull
    from sklearn.preprocessing import LabelEncoder

    adata = extract_adata_if_sdata(adata, table_key=table_key)
    assert_categorical_obs(adata, key=cluster_key)
    assert_spatial_basis(adata, key=spatial_key)
    coordinates = np.asarray(on_host(adata.obsm[spatial_key]))
    clusters = adata.obs[cluster_key].values
    mode = RipleyStat(mode)

    N = coordinates.shape[0]
    hull = ConvexHull(coordinates)
    area = hull.volume
    if max_dist is None:
        max_dist = (area / 2) ** 0.5
    support = np.linspace(0, max_dist, n_steps)

    le = LabelEncoder().fit(clusters)
    cluster_idx = le.transform(clusters)
    n_cls = le.classes_.shape[0]
    obs_arr = np.empty((n_cls, n_steps))

    start = time.perf_counter()
    logg.info("Calculating Ripley's %s statistic for `%d` clusters and `%d` simulations", mode, n_cls, n_simulations)
    obs_rng, *sim_rngs = spawn_generators(shared_seed(seed), n_simulations + 1)  # one family for all ranks (pair tiles are summed)
    bins = support

    if mode == RipleyStat.L:
        code = _check_l_metric(metric)
        # all simulations first (host RNG stream identical to the reference: one generator per simulation), then ONE
        # GPU launch counts pairs for the observed clusters and every simulated pattern
        groups = [coordinates[cluster_idx == i, :].astype(np.float64, copy=False) for i in range(int(np.max(cluster_idx)) + 1)]
        from scipy.spatial import Delaunay

        deln = Delaunay(hull.points[hull.vertices])  # one triangulation of the hull for all simulations
        sims_pts = [_ppp(hull, 1, n_observations, rng=sim_rngs[i], deln=deln).reshape(-1, 2) for i in range(n_simulations)]
        rank, ws = world()
        counts = pair_counts(groups + sims_pts, support, metric=code, ctx=default_context(device), shard=(rank, ws))
        counts = all_reduce_sum(counts)
        sizes = np.array([len(g) for g in groups + sims_pts], dtype=np.int64)
        l_all = _l_from_counts(counts, sizes, N, area)
        obs_arr[: len(groups)] = l_all[: len(groups)]
        sims = l_all[len(groups) :].reshape(n_simulations, n_steps)
    else:
        counts = _f_g_counts(mode, coordinates, cluster_idx, hull, support, metric, n_neigh, n_simulations, n_observations, obs_rng,
                             sim_rngs, device)
        stats = _f_g_from_counts(counts)
        obs_arr[: counts.shape[0] - n_simulations] = stats[: counts.shape[0] - n_simulations]
        sims = stats[counts.shape[0] - n_simulations :]

    pvalues = np.ones((n_cls, len(bins)))
    for i in range(n_simulations):
        for j in range(obs_arr.shape[0]):
            pvalues[j] += sims[i] >= obs_arr[j]
    pvalues /= n_simulations + 1
    pvalues = np.minimum(pvalues, 1 - pvalues)

    obs_df = _reshape_res(obs_arr.T, columns=le.classes_, index=bins, var_name=cluster_key)
    sims_df = _reshape_res(sims.T, columns=np.arange(n_simulations), index=bins, var_name="simulations")
    res = {f"{mode}_stat": obs_df, "sims_stat": sims_df, "bins": bins, "pvalues": pvalues}

    if copy:
        logg.info("Finish (%.3fs)", time.perf_counter() - start)
        return res
    _save_data(adata, attr="uns", key=Key.uns.ripley(cluster_key, mode), data=res, time_start=start)
    return None


def _check_l_metric(metric: str) -> int:
    """The kernel code of an L metric; names ``KDTree`` does not take raise the reference's error."""
    from sklearn.neighbors import KDTree

    if metric not in KDTree.valid_metrics:  # same check and message as _ripley.py:213-214
        raise ValueError(f"Unsupported metric '{metric}'. Ripley's L supports {KDTree.valid_metrics}")
    return metric_code(metric)


def _l_from_counts(counts: np.ndarray, sizes: np.ndarray, n: int, area: float) -> np.ndarray:
    """K/L estimate of ``_l_function`` (``_ripley.py:224-227``) from two-point counts that include self pairs."""
    n_pairs = counts - sizes[:, None]
    intensity = n / area
    k_estimate = (n_pairs / n) / intensity
    return np.sqrt(k_estimate / np.pi)


def _kd_tree_euclidean(metric: str, n_neigh: Any, n_fit: int) -> bool:
    """Whether ``NearestNeighbors(metric=metric, n_neighbors=n_neigh).fit(X)`` with ``n_fit`` 2-D points searches with its
    kd_tree under the euclidean distance (sklearn's ``auto`` rule: ``n_neighbors < n_fit // 2``) and k fits the kernel.  Below
    that size sklearn runs brute force, whose distances come from a GEMM form with other last bits."""
    if metric not in _EUCLIDEAN or isinstance(n_neigh, bool) or not isinstance(n_neigh, (int, np.integer)):
        return False
    return 1 <= int(n_neigh) <= _NN_MAX_K and int(n_neigh) < n_fit // 2


def _knn_hist_host(ref: np.ndarray, qry: np.ndarray, metric: str, n_neigh: Any, k: Any, support: np.ndarray) -> np.ndarray:
    """The reference's search and histogram with scikit-learn (``_ripley.py:145-150, 162-169, 206-207``)."""
    from sklearn.neighbors import NearestNeighbors

    tree = NearestNeighbors(metric=metric, n_neighbors=n_neigh).fit(ref)
    distances, _ = tree.kneighbors(qry, n_neighbors=k)
    return np.histogram(distances.squeeze(), bins=support)[0]


def _f_g_plan(mode: RipleyStat, coordinates: np.ndarray, cluster_idx: np.ndarray, draws_obs: list[np.ndarray], draws_sim: list[np.ndarray],
              support: np.ndarray, metric: str, n_neigh: Any) -> tuple[np.ndarray, np.ndarray, list[tuple]]:
    """The histograms of F / G as one point pool and task list for ``nn_distance_hist``, and the rows left to the host.

    Row c < n_clusters is the observed statistic of cluster c, row n_clusters + i simulation i.  G: cluster c against every
    point outside it (the two ranges on either side of c in the cluster-sorted pool), simulation i: all N points against draw
    i (k = 1).  F: draw c (one per cluster) against cluster c, simulation i: the last cluster's draw against draw i (k = 1).
    Returns (pool, tasks, host) where host lists ``(row, ref, qry, k)`` for the rows the device does not take."""
    n_cls = len(draws_obs) if mode == RipleyStat.F else int(np.max(cluster_idx)) + 1
    order = np.argsort(cluster_idx, kind="stable")
    ptr = np.zeros(n_cls + 1, dtype=np.int64)
    ptr[1:] = np.cumsum(np.bincount(cluster_idx, minlength=n_cls)[:n_cls])
    N = coordinates.shape[0]
    planar = coordinates.ndim == 2 and coordinates.shape[1] == 2
    ok_support = support.size >= 2 and bool(np.all(np.isfinite(support))) and bool(np.all(np.diff(support) >= 0))
    blocks = [np.asarray(coordinates, dtype=np.float64)[order]] if planar else []
    off = N
    draw_ptr = []
    for d in list(draws_obs) + list(draws_sim):
        planar_d = d.ndim == 2 and d.shape[1] == 2
        draw_ptr.append((off, off + d.shape[0]) if planar_d else None)
        if planar and planar_d:
            blocks.append(np.asarray(d, dtype=np.float64))
            off += d.shape[0]
    n_obs_draws = len(draws_obs)
    tasks: list[tuple[int, ...]] = []
    host: list[tuple] = []

    def add(row, ref_rng, qry_rngs, sets, k):
        """``sets()`` gives the (reference, query) arrays of the host call; built only for a row the device does not take."""
        ok = planar and ok_support and ref_rng is not None and all(q is not None for q in qry_rngs)
        if ok and sum(q[1] - q[0] for q in qry_rngs) > 0 and _kd_tree_euclidean(metric, n_neigh, int(ref_rng[1] - ref_rng[0])):
            tasks.extend((ref_rng[0], ref_rng[1], q[0], q[1], int(k), row) for q in qry_rngs if q[1] > q[0])
        else:
            host.append((row, *sets(), k))

    for c in range(n_cls):
        if mode == RipleyStat.F:
            add(c, (ptr[c], ptr[c + 1]), [draw_ptr[c]], lambda c=c: (coordinates[cluster_idx == c, :], draws_obs[c]), n_neigh)
        else:
            add(c, (ptr[c], ptr[c + 1]), [(0, ptr[c]), (ptr[c + 1], N)],
                lambda c=c: (coordinates[cluster_idx == c, :], coordinates[cluster_idx != c, :]), n_neigh)
    for i, d in enumerate(draws_sim):
        if mode == RipleyStat.F:
            add(n_cls + i, draw_ptr[n_obs_draws + i], [draw_ptr[n_obs_draws - 1]], lambda d=d: (d, draws_obs[-1]), 1)
        else:
            add(n_cls + i, draw_ptr[n_obs_draws + i], [(0, N)], lambda d=d: (d, coordinates), 1)
    pool = np.concatenate(blocks) if blocks else np.zeros((0, 2))
    return pool, np.asarray(tasks, dtype=np.int64).reshape(-1, 6), host


def _f_g_counts(mode: RipleyStat, coordinates: np.ndarray, cluster_idx: np.ndarray, hull, support: np.ndarray, metric: str, n_neigh: Any,
                n_simulations: int, n_observations: int, obs_rng: np.random.Generator, sim_rngs: list, device: int | None) -> np.ndarray:
    """int64 (n_clusters + n_simulations, n_steps - 1) histogram counts of F or G: every draw first (in the reference's RNG
    order: F's observed draws from ``obs_rng`` in cluster order, one generator per simulation), then ONE device call for the
    sets scikit-learn searches with its kd_tree, and scikit-learn for the rest in row order."""
    from scipy.spatial import Delaunay

    deln = Delaunay(hull.points[hull.vertices])  # the triangulation _ppp would build on every call
    n_cls = int(np.max(cluster_idx)) + 1
    draws_obs = [_ppp(hull, 1, n_observations, rng=obs_rng, deln=deln) for _ in range(n_cls)] if mode == RipleyStat.F else []
    draws_sim = [_ppp(hull, 1, n_observations, rng=sim_rngs[i], deln=deln) for i in range(n_simulations)]
    pool, tasks, host = _f_g_plan(mode, coordinates, cluster_idx, draws_obs, draws_sim, support, metric, n_neigh)
    counts = np.zeros((n_cls + n_simulations, max(len(support) - 1, 0)), dtype=np.int64)
    if tasks.shape[0]:
        rank, ws = world()
        counts = all_reduce_sum(nn_distance_hist(pool, tasks, support, counts.shape[0], ctx=default_context(device), shard=(rank, ws)))
    for row, ref, qry, k in host:
        counts[row] = _knn_hist_host(ref, qry, metric, n_neigh, k, support)
    return counts


def _f_g_from_counts(counts: np.ndarray) -> np.ndarray:
    """``_f_g_function`` (``_ripley.py:206-209``) of every row of histogram counts: [0, cumsum(counts) / counts.sum()]."""
    fracs = np.cumsum(counts, axis=-1) / counts.sum(axis=-1, keepdims=True)
    return np.concatenate((np.zeros(counts.shape[:-1] + (1,), dtype=float), fracs), axis=-1)


def _reshape_res(results: np.ndarray, columns, index: np.ndarray, var_name: str) -> pd.DataFrame:
    df = pd.DataFrame(results, columns=columns, index=index)
    df.index.set_names(["bins"], inplace=True)
    df = df.melt(var_name=var_name, value_name="stats", ignore_index=False)
    df[var_name] = df[var_name].astype("category")
    df.reset_index(inplace=True)
    return df


def _ppp(hull, n_simulations: int, n_observations: int, rng: np.random.Generator, deln=None) -> np.ndarray:
    """Poisson point process on the convex hull by rejection from its bounding box (``_ripley.py:230-271``): one
    ``rng.uniform`` draw for x then one for y per candidate, accepted if inside the hull.  The draw order is part of the
    result.  The reference draws and tests one candidate at a time in Python; here candidates are drawn in blocks
    (``low + (high - low) * rng.random()`` is ``rng.uniform(low, high)`` bit for bit), tested with one vectorised
    ``find_simplex`` call, and the generator is then put back to the exact position the scalar loop would have reached
    (PCG64 ``advance`` by two draws per consumed candidate), so both the points and every later draw are identical."""
    from scipy.spatial import Delaunay

    vxs = hull.points[hull.vertices]
    if deln is None:
        deln = Delaunay(vxs)
    bbox = np.array([*vxs.min(0), *vxs.max(0)])
    wx, wy = bbox[2] - bbox[0], bbox[3] - bbox[1]
    result = np.empty((n_simulations, n_observations, 2))
    exact_rewind = type(rng.bit_generator).__name__ == "PCG64"
    for i_sim in range(n_simulations):
        if not exact_rewind:  # unknown bit generator: the reference's scalar loop
            i_obs = 0
            while i_obs < n_observations:
                x, y = rng.uniform(bbox[0], bbox[2]), rng.uniform(bbox[1], bbox[3])
                if deln.find_simplex((x, y)) >= 0:
                    result[i_sim, i_obs] = (x, y)
                    i_obs += 1
            continue
        got = 0
        while got < n_observations:
            k = max(64, int((n_observations - got) * 1.5) + 16)
            state = rng.bit_generator.state
            u = rng.random(2 * k)
            pts = np.stack([bbox[0] + wx * u[0::2], bbox[1] + wy * u[1::2]], axis=1)
            ok = np.flatnonzero(deln.find_simplex(pts) >= 0)
            take = min(ok.size, n_observations - got)
            result[i_sim, got : got + take] = pts[ok[:take]]
            got += take
            if got >= n_observations and take > 0:
                used = int(ok[take - 1]) + 1  # candidates the scalar loop would have drawn in this block
                if used < k:
                    rng.bit_generator.state = state
                    rng.bit_generator.advance(2 * used)
    return result.squeeze()
