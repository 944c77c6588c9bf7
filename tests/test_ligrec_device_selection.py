"""Host logic of ligrec / sepal on a device-resident expression matrix (no GPU, no library call): the observed-statistics
specification the device kernel follows (a Kahan group mean equal to pandas' bit for bit), the selection ligrec builds from
var names and obs alone (equal to the host path's frame), and the description of a device X for the gather call."""

from __future__ import annotations

import numpy as np
import pandas as pd
import pytest

import squidpy_b200 as sq
from squidpy_b200._device import device_matrix, matrix_args
from squidpy_b200.gr import _ligrec
from tests.test_device_input_parsing import FakeDev, FakeSparse


def kahan_group_mean(x: np.ndarray, codes: np.ndarray, n_cls: int) -> np.ndarray:
    """What ``ligrec_observed_kernel`` computes: per (cluster, gene) a Kahan sum in cell order whose NaN compensation is reset,
    divided by the count."""
    s = np.zeros((n_cls, x.shape[1]))
    comp = np.zeros_like(s)
    for c in range(x.shape[0]):
        k = codes[c]
        y = x[c] - comp[k]
        t = s[k] + y
        with np.errstate(invalid="ignore"):
            cp = (t - s[k]) - y
        comp[k] = np.where(np.isnan(cp), 0.0, cp)
        s[k] = t
    return s / np.bincount(codes, minlength=n_cls)[:, None].astype(np.float64)


def _adversarial(rng, n=400, g=12, n_cls=5):
    mag = 10.0 ** rng.integers(-8, 8, (n, g))
    x = rng.standard_normal((n, g)) * mag
    x[rng.random((n, g)) < 0.3] = 0.0
    x[rng.random((n, g)) < 0.05] = np.nan  # becomes 0 through fillna
    x[5, 1], x[9, 1] = np.inf, -np.inf  # one gene with both infinities
    x[7, 2] = np.inf
    x[11, 3] = -np.inf
    x[:, 4] = np.tile([1e16, 1.0, -1e16, 3.0], n // 4)  # cancellation
    codes = rng.integers(0, n_cls - 1, n)
    codes[n // 2] = n_cls - 1  # a one-cell cluster
    return x, codes, n_cls


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_kahan_restatement_equals_pandas_group_mean(seed):
    x, codes, n_cls = _adversarial(np.random.default_rng(seed))
    df = pd.DataFrame(x, columns=list(range(x.shape[1]))).fillna(0.0)
    df["clusters"] = pd.Categorical(codes, categories=list(range(n_cls)))
    groups = df.groupby("clusters", observed=True)
    expected = groups.mean().values
    got = kahan_group_mean(np.nan_to_num(x, nan=0.0, posinf=np.inf, neginf=-np.inf), codes, n_cls)
    np.testing.assert_array_equal(got, expected)
    for thr in (0.0, 0.01, 0.3, 1.0):
        mask = groups.apply(lambda c: ((c > 0).astype(np.int64).sum() / len(c)) >= thr).values
        filled = df.drop(columns="clusters").to_numpy()
        npos = np.stack([(filled[codes == k] > 0).sum(0) for k in range(n_cls)]).astype(np.int64)
        sizes = np.bincount(codes, minlength=n_cls).astype(np.float64)
        np.testing.assert_array_equal((npos / sizes[:, None]) >= thr, mask)


def _names_case(rng, n=300):
    base = ["Cd4", "CD4", "Il2", "IL2RA", "Il2rb", "Il2rg", "Tgfb1", "tgfb1", "Ccl5", "Ccr5", "Cxcl12", "Cxcr4", "Actb", "Gapdh"]
    x = rng.poisson(0.7, (n, len(base))).astype(np.float32) * rng.random((n, len(base))).astype(np.float32)
    x[rng.random(x.shape) < 0.02] = np.nan
    labels = rng.choice(["b", "a", "c", "d"], n)
    obs = pd.DataFrame({"cl": pd.Categorical(labels)}, index=[f"c{i}" for i in range(n)])
    inter = pd.DataFrame({"source": ["il2", "IL2", "cd4", "ccl5", "CXCL12", "tgfb1", "nope", "Il2_Il2ra", "Il2ra_Il2rb_Il2rg"],
                          "target": ["il2ra_il2rb", "IL2RB_IL2RG", "Ccr5", "CCR5", "cxcr4", "Actb_Gapdh", "Cd4", "Cxcr4", "Ccl5"],
                          "note": list("abcdefghi")})
    return x, obs, base, inter


def _host_call(monkeypatch, x, obs, names, inter, **kw):
    got = {}

    def fake(sub, inter_, clusters_, **_):
        got.update(sub=sub, inter_=inter_, clusters_=clusters_)
        return _ligrec.TempResult(np.zeros((inter_.shape[0], clusters_.shape[0])), np.zeros((inter_.shape[0], clusters_.shape[0])))

    monkeypatch.setattr(_ligrec, "ligrec_analysis", fake)
    monkeypatch.setattr(_ligrec, "default_context", lambda device=None: None)
    ad = sq.AnnDataLite(X=x, obs=obs, var=pd.DataFrame(index=names))
    res = sq.gr.ligrec(ad, "cl", interactions=inter, use_raw=False, copy=True, n_perms=10, **kw)
    return got, res


@pytest.mark.parametrize("policy", ["min", "all"])
@pytest.mark.parametrize("clusters", [None, ["a", "c"], [("d", "b"), ("b", "b")]])
@pytest.mark.parametrize("seed", [0, 1])
def test_selection_from_names_equals_host_frame(monkeypatch, policy, clusters, seed):
    x, obs, names, inter = _names_case(np.random.default_rng(seed))
    got, res = _host_call(monkeypatch, x, obs, names, inter.copy(), complex_policy=policy, clusters=clusters)
    filled = np.where(np.isnan(x), np.float32(0), x)
    calls = []

    def read_columns(pos):
        calls.append(pos)
        return np.ascontiguousarray(filled[:, pos])

    sel = _ligrec._select_by_names(sq.AnnDataLite(X=None, obs=obs, var=pd.DataFrame(index=names), shape=x.shape), pd.Index(names), "cl",
                                   inter.copy(), policy, 10, clusters, read_columns)
    sub = got["sub"]
    assert len(calls) == (1 if policy == "min" else 0)
    np.testing.assert_array_equal(sub.drop(columns="clusters").to_numpy(), filled[sel.rows][:, sel.gene_pos].astype(np.float32))
    assert list(sub.index) == [f"c{i}" for i in sel.rows]
    np.testing.assert_array_equal(np.asarray(sub["clusters"].values, dtype=np.int32), sel.codes)
    assert sel.n_cls == len(sub["clusters"].cat.categories)
    np.testing.assert_array_equal(got["inter_"], sel.inter_)
    np.testing.assert_array_equal(got["clusters_"], sel.clusters_)
    assert list(res["means"].index) == list(pd.MultiIndex.from_frame(sel.pairs))
    assert list(res["means"].columns) == sel.clusters
    assert list(res["metadata"]["note"]) == list(sel.inter["note"])


def test_selection_errors_match_host(monkeypatch):
    x, obs, names, _ = _names_case(np.random.default_rng(3))
    ad = sq.AnnDataLite(X=None, obs=obs, var=pd.DataFrame(index=names), shape=x.shape)
    with pytest.raises(ValueError, match="no interactions remain"):
        _ligrec._select_by_names(ad, pd.Index(names), "cl", [("zz", "yy")], "min", 10, None, None)
    with pytest.raises(ValueError, match="Invalid cluster"):
        _ligrec._select_by_names(ad, pd.Index(names), "cl", [("Cd4", "Ccr5")], "min", 10, ["a", "q"], None)


def test_device_matrix_description():
    d = matrix_args(device_matrix(FakeDev((4, 6), "<f2", strides=(2, 8))), (4, 6))
    assert (d.format, d.code, d.strides, d.nnz) == (0, 2, (1, 4), 0)
    csr = matrix_args(device_matrix(FakeSparse("csr", (4, 9), n_ptr=5, nnz=7, stream=3)), (4, 9))
    assert (csr.format, csr.indptr_bits, csr.index_bits, csr.nnz, csr.code, csr.stream) == (1, 64, 32, 7, 1, 3)
    assert (csr.x, csr.indptr, csr.indices) == (0x3000, 0x1000, 0x2000)
    csc = matrix_args(device_matrix(FakeSparse("csc", (9, 4), n_ptr=5, nnz=7)), (9, 4))
    assert csc.format == 2
    with pytest.raises(ValueError, match="shape"):
        matrix_args(device_matrix(FakeDev((4, 6))), (4, 7))
    with pytest.raises(ValueError, match="indptr"):
        matrix_args(device_matrix(FakeSparse("csr", (5, 9), n_ptr=5)), (5, 9))
    with pytest.raises(TypeError, match="dtype"):
        matrix_args(device_matrix(FakeDev((4, 6), "|b1")), (4, 6))
    bad = FakeSparse("csr", (4, 9))
    bad.indices = FakeDev((7,), "<f4", ptr=0x2000)
    with pytest.raises(TypeError, match="int32 or int64"):
        matrix_args(device_matrix(bad), (4, 9))
    short = FakeSparse("csr", (4, 9))
    short.data = FakeDev((6,), "<f8", ptr=0x3000)
    with pytest.raises(ValueError, match="contiguous"):
        matrix_args(device_matrix(short), (4, 9))
    with pytest.raises(ValueError, match="different producer streams"):
        s = FakeSparse("csr", (4, 9), stream=3)
        s.data = FakeDev((7,), "<f8", ptr=0x3000, stream=4)
        matrix_args(device_matrix(s), (4, 9))
