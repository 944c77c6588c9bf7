"""GPU parity of tl.sliding_window: ``sqb_window_ranges`` against the numpy restatement ``tests/windows_ref.py`` at 1 M
observations (edges hit exactly and one ulp to either side, in float64, float32 and int64, NaN coordinates, an empty
library), its argument checks, and ``sliding_window`` against the reference's golden frames and against itself with the
kernel replaced by the restatement."""

from __future__ import annotations

import os

import numpy as np
import pandas as pd
import pytest

import squidpy_b200 as sq
from squidpy_b200 import AnnDataLite
from squidpy_b200.tl import _sliding_window, window_ranges
from tests import windows_ref
from tests.golden.make_golden_sliding_window import CASES, COPY_FALSE, ERRORS, decode, make_adata
from tools import sliding_window_time as st

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sliding_window.npz")


@pytest.mark.parametrize("case", range(len(CASES)))
def test_frame_equals_reference_golden(case):
    g = np.load(GOLDEN)
    name, kw = CASES[case]
    df = sq.tl.sliding_window(make_adata(name, AnnDataLite), copy=True, **kw)
    pd.testing.assert_frame_equal(df, decode(g, f"case{case}"), check_exact=True)


@pytest.mark.parametrize("case", range(len(COPY_FALSE)))
def test_copy_false_writes_obs(case):
    g = np.load(GOLDEN)
    name, kw = COPY_FALSE[case]
    adata = make_adata(name, AnnDataLite)
    sq.tl.sliding_window(adata, **kw)
    pd.testing.assert_frame_equal(adata.obs, decode(g, f"inplace{case}"), check_exact=True)


@pytest.mark.parametrize("case", range(len(ERRORS)))
def test_errors_raise_reference_type_and_message(case):
    g = np.load(GOLDEN)
    name, kw = ERRORS[case]
    with pytest.raises(Exception) as info:
        sq.tl.sliding_window(make_adata(name, AnnDataLite), copy=True, **kw)
    assert (type(info.value).__name__, str(info.value)) == (str(g["error_types"][case]), str(g["error_messages"][case]))


def _edge_problem(dtype, n=1_000_000, seed=0):
    """4 interleaved libraries with 10 x 10 windows each (400 in all) plus an empty fifth library; every coordinate is an edge
    or one ulp (one unit) to either side of one, a few are NaN (float dtypes); library 3 has its x axis without windows."""
    rng = np.random.default_rng(seed)
    lib = rng.integers(0, 4, n).astype(np.int32)
    lib[rng.integers(0, n, 1000)] = -1
    xy = np.empty((n, 2), dtype=dtype)
    edge_off, starts, ends = [0], [], []
    for code in range(5):
        rows = np.flatnonzero(lib == code)
        for axis in (0, 1):
            lo = dtype(0.1 * code + 3.0 * axis) if dtype != np.int64 else dtype(-50 * code + 7 * axis)
            s, e = _sliding_window._axis_windows(lo, lo + dtype(1000), 110, 10, code == 2)
            if code == 4 or (code == 3 and axis == 0):
                s, e = s[:0], e[:0]
            cmp_dt = np.result_type(dtype, s.dtype)
            edges = np.unique(np.concatenate([s, e]).astype(cmp_dt)) if s.size else np.array([lo], dtype=cmp_dt)
            if dtype == np.int64:
                vals = np.concatenate([edges - 1, edges, edges + 1])
            else:
                ev = edges.astype(dtype)
                vals = np.concatenate([np.nextafter(ev, dtype(-np.inf)), ev, np.nextafter(ev, dtype(np.inf))])
            xy[rows, axis] = rng.choice(vals, rows.size)
            starts.append(s), ends.append(e)
            edge_off.append(edge_off[-1] + s.size)
    if dtype != np.int64:
        xy[rng.integers(0, n, 500), rng.integers(0, 2, 500)] = np.nan
    kdt = np.int64 if dtype == np.int64 else np.float64
    return (xy.astype(kdt), lib, np.array(edge_off), np.concatenate(starts).astype(kdt), np.concatenate(ends).astype(kdt))


@pytest.mark.parametrize("dtype", [np.float64, np.float32, np.int64])
def test_kernel_equals_restatement_at_1m_edges(dtype):
    xy, lib, off, s, e = _edge_problem(dtype)
    got = window_ranges(xy, lib, off, s, e)
    np.testing.assert_array_equal(got, windows_ref.window_ranges(xy, lib, off, s, e))
    inside = (got[:, 0] <= got[:, 1]) & (got[:, 2] <= got[:, 3])
    assert not inside[(lib < 0) | (lib >= 3)].any()
    if dtype != np.int64:
        assert not inside[np.isnan(xy).any(axis=1)].any()


def test_empty_input():
    out = window_ranges(np.zeros((0, 2)), np.zeros(0, np.int32), np.array([0, 1, 2]), np.zeros(2), np.ones(2))
    assert out.shape == (0, 4)


@pytest.mark.parametrize("xy, lib, off, s, e, match", [
    (np.zeros((3, 2)), [0, 1, 0], [0, 1, 2], [0.0, 0.0], [1.0, 1.0], "outside"),
    (np.zeros((3, 2)), [0, -2, 0], [0, 1, 2], [0.0, 0.0], [1.0, 1.0], "outside"),
    (np.zeros((3, 2)), [0, 0, 0], [0, 2, 3], [1.0, 0.0, 0.0], [1.0, 1.0, 1.0], "decrease"),
    (np.zeros((3, 2)), [0, 0, 0], [0, 2, 3], [0.0, 1.0, 0.0], [2.0, 1.0, 1.0], "decrease"),
    (np.zeros((3, 2)), [0, 0, 0], [0, 2, 3], [0.0, np.nan, 0.0], [1.0, 2.0, 1.0], "NaN"),
    (np.zeros((3, 2)), [0, 0, 0], [1, 1, 2], [0.0, 0.0], [1.0, 1.0], "expected 0"),
    (np.zeros((3, 2)), [0, 0, 0], [0, 3, 2], [0.0, 0.0], [1.0, 1.0], "not a range"),
    (np.zeros((3, 2)), [0, 0], [0, 1, 2], [0.0, 0.0], [1.0, 1.0], "do not fit"),
])
def test_invalid_arguments_are_refused(xy, lib, off, s, e, match):
    with pytest.raises(ValueError, match=match):
        window_ranges(xy, np.array(lib), np.array(off), np.array(s), np.array(e))


def _restated(monkeypatch):
    monkeypatch.setattr(_sliding_window, "window_ranges", lambda xy, lib, off, s, e, *, ctx=None: windows_ref.window_ranges(xy, lib, off, s, e))


@pytest.mark.parametrize("name", list(st.SETTINGS))
def test_1m_cells_vs_restatement(monkeypatch, name):
    kw, n_libs, _ = st.SETTINGS[name]
    adata = st.make_adata(1_000_000, n_libs)
    got = sq.tl.sliding_window(adata, copy=True, **kw)
    _restated(monkeypatch)
    pd.testing.assert_frame_equal(got, sq.tl.sliding_window(adata, copy=True, **kw), check_exact=True)


def test_torch_cuda_coordinates_give_the_host_frame():
    import torch

    adata = st.make_adata(200_000, 3)
    kw = dict(window_size=700, overlap=100, library_key="library", copy=True)
    exp = sq.tl.sliding_window(adata, **kw)
    adata.obsm["spatial"] = torch.from_numpy(adata.obsm["spatial"]).cuda()
    pd.testing.assert_frame_equal(sq.tl.sliding_window(adata, **kw), exp, check_exact=True)
