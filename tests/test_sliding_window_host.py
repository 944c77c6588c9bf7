"""Host logic of tl.sliding_window, checked without a GPU: the restatement of the kernel against the reference's per-window
masks at every edge and one ulp to either side, the frame assembly (with the kernel replaced by that restatement) against
the reference's golden frames, its errors, and ``_calculate_window_corners`` against the reference's corner frames."""

from __future__ import annotations

import os

import numpy as np
import pandas as pd
import pytest

import squidpy_b200 as sq
from squidpy_b200 import AnnDataLite
from squidpy_b200.tl import _sliding_window
from tests import windows_ref
from tests.golden.make_golden_sliding_window import CASES, COPY_FALSE, CORNERS, ERRORS, decode, make_adata

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sliding_window.npz")


@pytest.fixture()
def host_kernel(monkeypatch):
    """``window_ranges`` replaced by the numpy restatement (and no CUDA context): every call the device would get."""
    calls = []

    def fake(xy, lib, edge_off, starts, ends, *, ctx=None):
        calls.append((np.asarray(xy).copy(), np.asarray(lib).copy(), np.asarray(edge_off).copy()))
        return windows_ref.window_ranges(xy, lib, edge_off, starts, ends)

    monkeypatch.setattr(_sliding_window, "window_ranges", fake)
    monkeypatch.setattr(_sliding_window, "default_context", lambda device=None: None)
    return calls


@pytest.mark.parametrize("case", range(len(CASES)))
def test_frame_equals_reference_golden(host_kernel, case):
    g = np.load(GOLDEN)
    name, kw = CASES[case]
    df = sq.tl.sliding_window(make_adata(name, AnnDataLite), copy=True, **kw)
    pd.testing.assert_frame_equal(df, decode(g, f"case{case}"), check_exact=True)
    assert len(host_kernel) == 1  # one device call for every library


@pytest.mark.parametrize("case", range(len(COPY_FALSE)))
def test_copy_false_writes_obs(host_kernel, case):
    g = np.load(GOLDEN)
    name, kw = COPY_FALSE[case]
    adata = make_adata(name, AnnDataLite)
    assert sq.tl.sliding_window(adata, **kw) is None
    pd.testing.assert_frame_equal(adata.obs, decode(g, f"inplace{case}"), check_exact=True)


@pytest.mark.parametrize("case", range(len(ERRORS)))
def test_errors_raise_reference_type_and_message(host_kernel, case):
    g = np.load(GOLDEN)
    name, kw = ERRORS[case]
    with pytest.raises(Exception) as info:
        sq.tl.sliding_window(make_adata(name, AnnDataLite), copy=True, **kw)
    assert type(info.value).__name__ == str(g["error_types"][case])
    assert str(info.value) == str(g["error_messages"][case])


def test_existing_key_is_overwritten_with_a_warning(host_kernel, caplog):
    adata = make_adata("libs_full", AnnDataLite)
    with caplog.at_level("WARNING", logger="squidpy_b200"):
        sq.tl.sliding_window(adata, window_size=2, library_key="lib", sliding_window_key="old")
    assert "Overwriting existing column 'old' in adata.obs." in caplog.text


def test_device_coordinates_are_read_on_the_host(host_kernel):
    torch = pytest.importorskip("torch")
    adata = make_adata("float32", AnnDataLite)
    exp = sq.tl.sliding_window(adata, window_size=2, overlap=1, library_key="lib", copy=True)
    adata.obsm["spatial"] = torch.from_numpy(adata.obsm["spatial"])
    pd.testing.assert_frame_equal(sq.tl.sliding_window(adata, window_size=2, overlap=1, library_key="lib", copy=True), exp, check_exact=True)


def _reference_masks(x, y, xs, xe, ys, ye):
    """The reference's loop (:130-143) over the windows of the product xs x ys: one mask per window, numpy's comparisons."""
    masks = []
    for i in range(xs.size):
        for j in range(ys.size):
            e = np.result_type(xs.dtype, xe.dtype, ys.dtype, ye.dtype)  # one row of iterrows: the common dtype of its edges
            masks.append((x >= e.type(xs[i])) & (x <= e.type(xe[i])) & (y >= e.type(ys[j])) & (y <= e.type(ye[j])))
    return np.stack(masks, 1) if masks else np.zeros((x.size, 0), dtype=bool)


@pytest.mark.parametrize("dtype", [np.float64, np.float32, np.int64])
@pytest.mark.parametrize("overlap, drop", [(0, False), (0, True), (3, False), (3, True)])
def test_restatement_equals_reference_masks_next_to_every_edge(dtype, overlap, drop):
    rng = np.random.default_rng(overlap + drop)
    lo = dtype(0.1) if dtype != np.int64 else dtype(-7)
    xs, xe, ys, ye = (*_sliding_window._axis_windows(lo, dtype(61), 7, overlap, drop), *_sliding_window._axis_windows(lo, dtype(44), 7, overlap, drop))
    edges = np.unique(np.concatenate([xs, xe, ys, ye]).astype(dtype))
    if dtype == np.int64:
        vals = np.concatenate([edges - 1, edges, edges + 1])
    else:
        vals = np.concatenate([np.nextafter(edges, dtype(-np.inf)), edges, np.nextafter(edges, dtype(np.inf))])
    x, y = rng.choice(vals, 3000).astype(dtype), rng.choice(vals, 3000).astype(dtype)
    e = np.result_type(xs.dtype, xe.dtype, ys.dtype, ye.dtype)
    kdt = _sliding_window._comparison_dtype(np.dtype(dtype), e)
    cast = [a.astype(e).astype(kdt) for a in (xs, ys, xe, ye)]
    got = windows_ref.window_ranges(np.stack([x.astype(np.result_type(dtype, e)), y.astype(np.result_type(dtype, e))], 1).astype(kdt),
                                    np.zeros(x.size, dtype=np.int32), np.array([0, xs.size, xs.size + ys.size]),
                                    np.concatenate(cast[:2]), np.concatenate(cast[2:]))
    np.testing.assert_array_equal(windows_ref.membership(got, xs.size, ys.size), _reference_masks(x, y, xs, xe, ys, ye))


@pytest.mark.parametrize("case", range(len(CORNERS)))
def test_window_corners_equal_reference_golden(case):
    g = np.load(GOLDEN)
    got = _sliding_window._calculate_window_corners(*CORNERS[case])
    pd.testing.assert_frame_equal(got, decode(g, f"corners{case}"), check_exact=True)


@pytest.mark.parametrize("overlap", [-1, 5, 6])
def test_window_corners_refuse_bad_overlap(overlap):
    with pytest.raises(ValueError, match="Overlap must be"):
        _sliding_window._calculate_window_corners(0, 10, 0, 10, 5, overlap)
