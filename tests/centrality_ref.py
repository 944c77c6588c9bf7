"""numpy / scipy restatement of ``sqb_centrality_scores`` (``csrc/centrality.cu``): the canonical undirected graph, the
integer counts per cluster and the local clustering coefficients.  Pinned to networkx and to the reference's golden output
by ``tests/test_centrality_host.py``; the GPU tests compare the kernels with it bit for bit."""

from __future__ import annotations

import numpy as np
import scipy.sparse as sp

from squidpy_b200.gr._nhood import CentralityCounts


def canonical(conn) -> sp.csr_matrix:
    """``A + Aᵀ`` with values summed in A's dtype, diagonal and zero sums dropped, as a sorted boolean CSR.  Per pair
    {i, j}: A's entries (i, j) in storage order, then Aᵀ's (A's entries (j, i)), each summed on its own, then the two sums."""
    a = conn if sp.issparse(conn) and conn.format in ("csr", "csc") else sp.csr_matrix(conn)
    n = a.shape[0]
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(a.indptr))
    cols = a.indices.astype(np.int64)
    off = rows != cols
    rows, cols, vals = rows[off], cols[off], a.data[off]
    # records (row, col, from_transpose, value), both directions, stable in storage order
    r = np.concatenate([rows, cols])
    c = np.concatenate([cols, rows])
    d = np.concatenate([np.zeros(rows.size, np.int64), np.ones(rows.size, np.int64)])
    v = np.concatenate([vals, vals])
    order = np.lexsort((np.arange(r.size), d, c, r))
    r, c, d, v = r[order], c[order], d[order], v[order]
    if r.size == 0:
        return sp.csr_matrix((n, n), dtype=bool)
    key = (r * n + c) * 2 + d
    head = np.flatnonzero(np.concatenate([[True], key[1:] != key[:-1]]))
    reduce = np.logical_or.reduceat if v.dtype == np.bool_ else np.add.reduceat
    part = reduce(v, head, dtype=v.dtype)  # one sum per (pair, direction) in A's dtype, sequential within
    pr, pc, pd = r[head], c[head], d[head]
    pair_head = np.concatenate([[True], (pr[1:] != pr[:-1]) | (pc[1:] != pc[:-1])])
    starts = np.flatnonzero(pair_head)
    total = part[starts].copy()
    second = np.flatnonzero(~pair_head)  # the transpose's sum of a pair that has both
    if v.dtype == np.bool_:
        total[np.searchsorted(starts, second, side="right") - 1] |= part[second]
    else:
        with np.errstate(over="ignore"):
            idx = np.searchsorted(starts, second, side="right") - 1
            total[idx] = total[idx] + part[second]
    keep = total != 0
    kr, kc = pr[starts][keep], pc[starts][keep]
    g = sp.csr_matrix((np.ones(kr.size, dtype=bool), (kr, kc)), shape=(n, n))
    g.sort_indices()
    return g


def counts(conn, codes, n_cls: int) -> CentralityCounts:
    """Every measure of ``sqb_centrality_scores``: |N(S) \\ S| and the summed hop distances per cluster (scipy's BFS from
    each group), the clustering coefficients, and the BFS depth."""
    from scipy.sparse.csgraph import dijkstra

    g = canonical(conn)
    codes = np.asarray(codes, dtype=np.int64)
    n = g.shape[0]
    rows = np.repeat(np.arange(n), np.diff(g.indptr))
    cols = g.indices.astype(np.int64)
    # degree: distinct (v, cluster of a neighbour) with v outside that cluster
    lab = codes[cols]
    m = (lab >= 0) & (lab != codes[rows])
    pairs = np.unique(rows[m] * max(n_cls, 1) + lab[m])
    reach1 = np.bincount(pairs % max(n_cls, 1), minlength=n_cls).astype(np.int64)
    dist = np.zeros(n_cls, dtype=np.int64)
    levels = 0
    for k in range(n_cls):
        src = np.flatnonzero(codes == k)
        if src.size == 0:
            continue
        dk = dijkstra(g, directed=False, unweighted=True, indices=src, min_only=True)
        fin = np.isfinite(dk)
        dist[k] = int(dk[fin].astype(np.int64).sum())
        levels = max(levels, int(dk[fin].max()))
    # clustering: 2 T(v) = sum over neighbours u of |N(u) ∩ N(v)| = ((A A) ∘ A) 1
    a = g.astype(np.int64)
    t2 = np.asarray((a @ a).multiply(a).sum(axis=1)).ravel().astype(np.int64)
    k = np.diff(g.indptr).astype(np.int64)
    cc = np.zeros(n, dtype=np.float64)
    ok = k >= 2
    cc[ok] = t2[ok] / (k[ok] * (k[ok] - 1))
    return CentralityCounts(reach1, dist, cc, levels)
