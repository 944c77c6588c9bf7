"""numpy / scipy restatement of the niche embeddings of ``csrc/niche.cu`` (test only).

* ``profile``: P_1 = A Y over the canonical graph (duplicates summed in A's dtype, ascending columns), P_k = A P_{k-1} in float64
  (scipy's csr @ dense adds each row's products in storage order); per hop the proportions with a sequential row total
  (NaN skipped, a NaN quotient -> 0); then the hop weights.
* ``utag``: the reference's own expression, ``normalize(A, "l1", axis=1) @ X``.
* ``cellcharter``: the reference's hop recursion (``_setdiag`` / ``_hop`` / ``_normalize``) on scipy, with one change the
  device makes: hop k >= 2 is put in ascending column order before it is normalised and applied, so its float64 sums run
  over ascending columns instead of scipy's non-canonical order.
"""

from __future__ import annotations

import numpy as np
import scipy.sparse as sp


def canonical(A) -> sp.csr_matrix:
    A = sp.csr_matrix(A, copy=True)
    A.sum_duplicates()
    return A


def profile(A, codes, n_cls, distance=1, weights=None, abs_nhood=False) -> np.ndarray:
    A = canonical(A).astype(np.float64)
    codes = np.asarray(codes)
    Y = np.zeros((len(codes), n_cls))
    ok = codes >= 0
    Y[np.flatnonzero(ok), codes[ok]] = 1.0
    P = A @ Y
    hops = [P]
    for _ in range(1, max(distance, 1)):
        P = A @ P
        hops.append(P)

    def share(P):
        if abs_nhood:
            return P
        t = np.nancumsum(P, axis=1)[:, -1] if P.shape[1] else np.zeros(P.shape[0])
        with np.errstate(divide="ignore", invalid="ignore"):
            q = P / t[:, None]
        q[np.isnan(q)] = 0.0
        return q

    if distance <= 1:
        return share(hops[0])
    w = [1.0] * distance if weights is None else list(weights)
    if len(w) < distance:
        w = w + [w[-1]] * (distance - len(w))
    out = w[0] * share(hops[0])
    for k in range(1, distance):
        out = out + w[k] * share(hops[k])
    return out if abs_nhood else out / sum(w)


def utag(A, X) -> np.ndarray:
    from sklearn.preprocessing import normalize

    out = normalize(A, norm="l1", axis=1) @ X
    return out.toarray() if sp.issparse(out) else np.asarray(out)


def _setdiag(A, value):
    A = A.tolil()
    A.setdiag(value)
    A = A.tocsr()
    if value == 0:
        A.eliminate_zeros()
    return A


def _normalize(H):
    deg = np.array(np.sum(H, axis=1)).squeeze(axis=1)
    with np.errstate(divide="ignore"):
        dinv = 1 / deg
    dinv[dinv == float("inf")] = 0
    return sp.spdiags(dinv, 0, len(dinv), len(dinv)) * H


def _aggregate(N, X, aggregation):
    if aggregation == "mean":
        out = N @ X
        return out.toarray() if sp.issparse(out) else np.asarray(out)
    Xd = X.toarray() if sp.issparse(X) else np.asarray(X)
    mean = N @ Xd
    return N @ (Xd * Xd) - mean * mean


def hops(A, distance) -> list[sp.csr_matrix]:
    """hop_1 .. hop_distance as the reference builds them, each with sorted indices."""
    A = canonical(A)
    H = _setdiag(A, 0)
    V = _setdiag(A.copy(), 1)
    out = [H]
    for _ in range(2, distance + 1):
        H = H @ A
        H = H > V
        V = V + H
        H = sp.csr_matrix(H)
        H.sort_indices()
        out.append(H)
    return out


def cellcharter(A, X, distance, aggregation="mean") -> tuple[np.ndarray, list[int]]:
    hs = hops(A, distance)
    blocks = [X.toarray() if sp.issparse(X) else np.asarray(X)]
    for k, H in enumerate(hs):
        N = _normalize(H)
        if k > 0:  # ascending columns, as the device takes hop k >= 2
            N = sp.csr_matrix(N)
            N.sort_indices()
        blocks.append(_aggregate(N, X, aggregation))
    dtype = np.result_type(*[b.dtype for b in blocks])
    return np.hstack([b.astype(dtype) for b in blocks]), [int(H.nnz) for H in hs]
