"""``ripley`` — drop-in for ``squidpy.gr.ripley`` (``src/squidpy/gr/_ripley.py:27-194``).

Mode ``L``: the expensive step — cumulative ordered-pair counts per cluster, ``KDTree.two_point_correlation`` in the
reference (:218-223) — runs on the H100 (``sqb_pair_counts_f64``: float64, bit-identical counts), for the observed
clusters and for all Poisson-point-process simulations in ONE launch.  Modes ``F``/``G`` need only 1-/2-nearest
neighbour distances of ~1000 points and stay on the host with scikit-learn, like in the reference; so do the convex
hull, the rejection-sampled simulations (they must consume numpy's RNG stream exactly) and the long-format reshaping.
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
from .._rng import spawn_generators
from .._validators import assert_categorical_obs, assert_spatial_basis, extract_adata_if_sdata
from ._utils import _save_data, logg

__all__ = ["ripley", "pair_counts"]


def pair_counts(groups: list[np.ndarray], support: np.ndarray, *, ctx: Context | None = None, shard: tuple[int, int] = (0, 1)) -> np.ndarray:
    """For every point set in ``groups`` (each (m, 2) float64): int64 (len(groups), S) counts of ordered pairs,
    self pairs included, with ``sqrt(dx^2 + dy^2) <= support[s]`` — i.e. ``KDTree(p).two_point_correlation(p, support)``."""
    lib = load()
    ctx = ctx or default_context()
    support = np.ascontiguousarray(support, dtype=np.float64)
    ptr = np.zeros(len(groups) + 1, dtype=np.int64)
    ptr[1:] = np.cumsum([len(g) for g in groups])
    pts = np.ascontiguousarray(np.concatenate([np.asarray(g, dtype=np.float64).reshape(-1, 2) for g in groups], axis=0)) if ptr[-1] else np.zeros((1, 2))
    out = np.empty((len(groups), support.size), dtype=np.int64)
    check(lib.sqb_pair_counts_f64(ctx.handle, pts.ctypes.data, ptr.ctypes.data, len(groups), support.ctypes.data, support.size,
                                  int(shard[0]), int(shard[1]), out.ctypes.data))
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
    from sklearn.neighbors import NearestNeighbors
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
        _check_l_metric(metric)
        # all simulations first (host RNG stream identical to the reference: one generator per simulation), then ONE
        # GPU launch counts pairs for the observed clusters and every simulated pattern
        groups = [coordinates[cluster_idx == i, :].astype(np.float64, copy=False) for i in range(int(np.max(cluster_idx)) + 1)]
        from scipy.spatial import Delaunay

        deln = Delaunay(hull.points[hull.vertices])  # one triangulation of the hull for all simulations
        sims_pts = [_ppp(hull, 1, n_observations, rng=sim_rngs[i], deln=deln).reshape(-1, 2) for i in range(n_simulations)]
        rank, ws = world()
        counts = pair_counts(groups + sims_pts, support, ctx=default_context(device), shard=(rank, ws))
        counts = all_reduce_sum(counts)
        sizes = np.array([len(g) for g in groups + sims_pts], dtype=np.int64)
        l_all = _l_from_counts(counts, sizes, N, area)
        obs_arr[: len(groups)] = l_all[: len(groups)]
        sims = l_all[len(groups) :].reshape(n_simulations, n_steps)
    else:
        random = None
        for i in np.arange(np.max(cluster_idx) + 1):
            coord_c = coordinates[cluster_idx == i, :]
            if mode == RipleyStat.F:
                random = _ppp(hull, n_simulations=1, n_observations=n_observations, rng=obs_rng)
                tree_c = NearestNeighbors(metric=metric, n_neighbors=n_neigh).fit(coord_c)
                distances, _ = tree_c.kneighbors(random, n_neighbors=n_neigh)
            else:
                tree_c = NearestNeighbors(metric=metric, n_neighbors=n_neigh).fit(coord_c)
                distances, _ = tree_c.kneighbors(coordinates[cluster_idx != i, :], n_neighbors=n_neigh)
            bins, obs_stats = _f_g_function(distances.squeeze(), support)
            obs_arr[i] = obs_stats
        sims = np.empty((n_simulations, len(bins)))
        for i in range(n_simulations):
            random_i = _ppp(hull, n_simulations=1, n_observations=n_observations, rng=sim_rngs[i])
            tree_i = NearestNeighbors(metric=metric, n_neighbors=n_neigh).fit(random_i)
            if mode == RipleyStat.F:
                distances_i, _ = tree_i.kneighbors(random, n_neighbors=1)
            else:
                distances_i, _ = tree_i.kneighbors(coordinates, n_neighbors=1)
            _, sims[i] = _f_g_function(distances_i.squeeze(), support)

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


def _check_l_metric(metric: str) -> None:
    from sklearn.neighbors import KDTree

    if metric not in KDTree.valid_metrics:  # same check and message as _ripley.py:213-214
        raise ValueError(f"Unsupported metric '{metric}'. Ripley's L supports {KDTree.valid_metrics}")
    if metric not in ("euclidean", "l2", "minkowski", "p"):
        raise NotImplementedError(f"Ripley's L on the GPU implements the euclidean metric only, found `{metric}`.")


def _l_from_counts(counts: np.ndarray, sizes: np.ndarray, n: int, area: float) -> np.ndarray:
    """K/L estimate of ``_l_function`` (``_ripley.py:224-227``) from two-point counts that include self pairs."""
    n_pairs = counts - sizes[:, None]
    intensity = n / area
    k_estimate = (n_pairs / n) / intensity
    return np.sqrt(k_estimate / np.pi)


def _reshape_res(results: np.ndarray, columns, index: np.ndarray, var_name: str) -> pd.DataFrame:
    df = pd.DataFrame(results, columns=columns, index=index)
    df.index.set_names(["bins"], inplace=True)
    df = df.melt(var_name=var_name, value_name="stats", ignore_index=False)
    df[var_name] = df[var_name].astype("category")
    df.reset_index(inplace=True)
    return df


def _f_g_function(distances: np.ndarray, support: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    counts, bins = np.histogram(distances, bins=support)
    fracs = np.cumsum(counts) / counts.sum()
    return bins, np.concatenate((np.zeros((1,), dtype=float), fracs))


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
