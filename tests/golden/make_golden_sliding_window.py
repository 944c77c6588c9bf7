"""Generates tests/golden/sliding_window.npz: the UNMODIFIED reference ``tl.sliding_window`` (a squidpy source checkout,
``$SQUIDPY_REF``, through the stub-import loader ``oracle/_refload.py``) on fixtures that reach every branch of its window
assignment.  Only runnable where the reference tree exists; the output is committed.

    python tests/golden/make_golden_sliding_window.py

Fixtures (``fixture(name)``): an integer lattice with observations on every shared window edge and corner; float64 points on
``arange``'s own ``start + i * step`` edges and one ulp to either side of them; float32 coordinates in ``obsm``; int64
``globalX`` / ``globalY`` obs columns next to an ``obsm`` that must be ignored; 3-D ``obsm``; four interleaved libraries, one
of them a single point; NaN coordinates.  Frames are stored without pickles: column names, per column a kind (``category``
with codes, categories and the ordered flag; ``object_bool`` for object columns of ``True`` / ``False``; else the numpy
dtype), and the index.  Every error case stores the exception's type name and message.
"""

from __future__ import annotations

import importlib
import os
import sys
import types

import numpy as np
import pandas as pd

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.dirname(os.path.abspath(__file__))

# (fixture, kwargs); copy=True unless kwargs say otherwise
CASES = [
    ("lattice", dict(window_size=4)),
    ("lattice", dict(window_size=4, overlap=2)),
    ("lattice", dict(window_size=5, drop_partial_windows=False, overlap=3)),
    ("lattice", dict(window_size=5, overlap=2, drop_partial_windows=True)),
    ("lattice", dict(window_size=3, library_key="lib")),
    ("lattice", dict(window_size=3, overlap=1, library_key="lib", drop_partial_windows=True)),
    ("lattice", dict()),
    ("float64", dict(window_size=3)),
    ("float64", dict(window_size=3, overlap=1)),
    ("float64", dict(window_size=2, library_key="lib")),
    ("float64", dict(library_key="lib", overlap=1)),
    ("float32", dict(window_size=2)),
    ("float32", dict(window_size=2, overlap=1, library_key="lib")),
    ("int_obs", dict(window_size=250)),
    ("int_obs", dict(window_size=300, overlap=100, drop_partial_windows=True)),
    ("int_obs", dict(window_size=200, library_key="lib")),
    ("int_obs", dict()),
    ("spatial3d", dict(window_size=3, spatial_key="xyz")),
    ("spatial3d", dict(window_size=3, overlap=1, spatial_key="xyz", coord_columns=("cx", "cy"), sliding_window_key="sw")),
    ("libs", dict(window_size=2, overlap=1, library_key="lib")),
    ("libs", dict(window_size=3, overlap=2, library_key="lib", drop_partial_windows=True, sliding_window_key="win")),
    ("libs_full", dict(window_size=2, library_key="lib")),
    ("libs_full", dict(window_size=2, library_key="lib", coord_columns=("px", "py"), sliding_window_key="tile")),
    ("libs_full", dict(library_key="lib")),
    ("nan", dict(window_size=3, overlap=1)),
    ("nan", dict(window_size=3, overlap=1, library_key="lib", drop_partial_windows=True)),
]

# (fixture, kwargs) written back into obs (copy=False); the stored frame is obs afterwards
COPY_FALSE = [
    ("lattice", dict(window_size=4, library_key="lib")),
    ("int_obs", dict(window_size=300, overlap=100)),
    ("libs_full", dict(window_size=2, library_key="lib", sliding_window_key="old")),
]

# _calculate_window_corners(min_x, max_x, min_y, max_y, window_size, overlap, drop_partial_windows)
CORNERS = [
    (0.1, 20.3, np.float32(-2.5), np.float32(9.0), 5, 0, False),
    (0.1, 20.3, np.float32(-2.5), np.float32(9.0), 5, 2, True),
    (np.int64(-3), np.int64(17), np.int64(4), np.int64(30), 5, 0, True),
    (np.int64(-3), np.int64(17), np.int64(4), np.int64(30), 5, 4, False),
    (np.int64(0), np.int64(12), 0.5, 7.0, 4, 1, False),
    (2.0, 2.0, 0.0, 10.0, 5, 0, False),
    (0.0, 3.0, 0.0, 3.0, 5, 0, True),
    (0.0, 3.0, 0.0, 3.0, 5, 2, False),
]

# (fixture, kwargs) the reference rejects
ERRORS = [
    ("lattice", dict(window_size=4, overlap=-1)),
    ("lattice", dict(window_size=0)),
    ("lattice", dict(window_size=-3, overlap=1)),
    ("lattice", dict(window_size=4, library_key="nope")),
    ("lattice", dict(window_size=4, overlap=4)),
    ("lattice", dict(window_size=4, overlap=7, library_key="lib")),
    ("lattice", dict(window_size=4, spatial_key="nope")),
    ("lattice", dict(window_size=4, drop_partial_windows=True)),
    ("nan", dict(window_size=3)),
    ("nan_lib", dict(window_size=3, library_key="lib")),
    ("nan_lib", dict(window_size=3, overlap=1, library_key="lib")),
    ("libs", dict(window_size=2, library_key="lib")),
    ("single", dict(window_size=2)),
    ("single", dict(window_size=2, library_key="lib")),
]


def fixture(name: str) -> tuple[pd.DataFrame, dict]:
    """obs and obsm of the named fixture; obs names are not in row order."""
    rng = np.random.default_rng(sum(map(ord, name)))
    obsm: dict = {}
    cols: dict = {}
    if name == "lattice":  # every integer point of [0, 12] x [0, 9]: windows of 3, 4 or 5 share edges and corners with them
        gx, gy = np.meshgrid(np.arange(13), np.arange(10))
        xy = np.stack([gx.ravel(), gy.ravel()], 1).astype(np.float64)
        obsm["spatial"] = xy[rng.permutation(len(xy))]
        cols["lib"] = np.where(rng.random(len(xy)) < 0.5, "s0", "s1")
    elif name == "float64":  # arange's own edges start + i * step (start 0.1) and one ulp to either side of them
        e = np.concatenate([np.arange(0.1, 9.7, 1.0), np.arange(0.1, 9.7, 1.0) + 2, np.arange(0.1, 9.7, 1.0) + 3])
        v = np.concatenate([e, np.nextafter(e, -np.inf), np.nextafter(e, np.inf), [0.1, 9.7]])
        v = v[(v >= 0.1) & (v <= 9.7)]
        xy = np.stack([v, rng.permutation(v)], 1)
        obsm["spatial"] = xy
        cols["lib"] = np.where(np.arange(len(xy)) % 3 == 0, "b", "a")
    elif name == "float32":  # float64 edges from float32 minima (0.1 -> 0.10000000149...), float32 points on and next to them
        e = (np.float32(0.1) + np.arange(6, dtype=np.float64)).astype(np.float32)
        v = np.concatenate([e, np.nextafter(e, np.float32(-np.inf)), np.nextafter(e, np.float32(np.inf)), rng.random(40).astype(np.float32) * 5])
        v = v[(v >= np.float32(0.1)) & (v <= np.float32(5.3))]
        obsm["spatial"] = np.stack([v, rng.permutation(v)], 1).astype(np.float32)
        cols["lib"] = rng.choice(["l1", "l0"], len(v))
    elif name == "int_obs":  # int64 coordinates in obs; obsm["spatial"] is something else and must not be read
        x = np.concatenate([rng.integers(-500, 1500, 60), np.arange(-500, 1501, 100)])
        y = np.concatenate([rng.integers(20, 1020, 60), np.arange(20, 1021, 50)])
        cols["globalX"], cols["globalY"] = x.astype(np.int64), y.astype(np.int64)
        obsm["spatial"] = rng.random((len(x), 2)) * 1e6
        cols["lib"] = pd.Categorical(np.where(rng.random(len(x)) < 0.4, 7, 3))
    elif name == "spatial3d":
        gx, gy = np.meshgrid(np.arange(8), np.arange(7))
        obsm["xyz"] = np.stack([gx.ravel(), gy.ravel(), rng.random(gx.size)], 1)
    elif name in ("libs", "libs_full"):  # four interleaved libraries; in "libs" library "solo" is a single point
        n = 80
        lib = rng.choice(["q", "p", "solo", "r"] if name == "libs" else ["q", "p", "r", "t"], n, p=[0.3, 0.3, 0.1, 0.3])
        if name == "libs":
            lib[lib == "solo"] = "p"
            lib[17] = "solo"
        xy = rng.integers(0, 9, (n, 2)).astype(np.float64) + (lib == "r")[:, None] * 100.0
        obsm["spatial"] = xy
        cols["lib"] = pd.Categorical(lib, categories=["t", "solo", "r", "q", "p"])
        cols["px"], cols["py"] = xy[:, 0] * 2, xy[:, 1] - 1
        cols["old"] = np.arange(n)
    elif name in ("nan", "nan_lib"):
        xy = rng.integers(0, 10, (50, 2)).astype(np.float64)
        xy[[3, 30], [0, 1]] = np.nan
        obsm["spatial"] = xy
        lib = np.where(np.arange(50) % 2 == 0, "u", "v").astype(object)
        if name == "nan_lib":
            xy[[3, 30], [0, 1]] = 1.0
            lib[10] = np.nan
        cols["lib"] = lib
    elif name == "single":
        obsm["spatial"] = np.array([[2.0, 3.0]])
        cols["lib"] = ["only"]
    else:
        raise ValueError(name)
    n = len(next(iter(obsm.values())))
    names = [f"obs{int(i)}" for i in rng.permutation(n)]
    return pd.DataFrame(cols, index=pd.Index(names)), obsm


class RowAnnData:
    """The AnnData surface the reference's sliding_window reads: obs, obsm, len and copy."""

    def __init__(self, obs, obsm):
        self.obs = obs
        self.obsm = dict(obsm)

    def __len__(self):
        return len(self.obs)

    def copy(self):
        return RowAnnData(self.obs.copy(), {k: v.copy() for k, v in self.obsm.items()})


def make_adata(name: str, cls=None):
    obs, obsm = fixture(name)
    if cls is None:
        return RowAnnData(obs, obsm)
    return cls(obs=obs, obsm=obsm, shape=(len(obs), 0))


def load_reference():
    from oracle import _refload

    _refload.load()
    m = types.ModuleType("squidpy.tl")
    m.__path__ = [f"{_refload.REF_SRC}/squidpy/tl"]  # type: ignore[attr-defined]
    sys.modules["squidpy.tl"] = m
    return importlib.import_module("squidpy.tl._sliding_window")


def encode(df: pd.DataFrame, prefix: str) -> dict[str, np.ndarray]:
    """A frame as plain arrays: column names, per column its kind and values, the index."""
    out = {f"{prefix}_columns": np.array([str(c) for c in df.columns]), f"{prefix}_index": np.array([str(i) for i in df.index]),
           f"{prefix}_index_dtype": np.array(str(df.index.dtype))}
    kinds = []
    for j in range(df.shape[1]):
        s = df.iloc[:, j]
        if isinstance(s.dtype, pd.CategoricalDtype):
            kinds.append("category_ordered" if s.cat.ordered else "category")
            out[f"{prefix}_c{j}_codes"] = np.asarray(s.cat.codes, dtype=np.int64)
            out[f"{prefix}_c{j}_categories"] = np.array(s.cat.categories.tolist())
        elif s.dtype == object and all(v is True or v is False for v in s):
            kinds.append("object_bool")
            out[f"{prefix}_c{j}"] = s.to_numpy().astype(bool)
        else:
            kinds.append(str(s.dtype))
            v = s.to_numpy()
            out[f"{prefix}_c{j}"] = np.array(v.tolist()) if v.dtype == object else v  # strings as a unicode array
    out[f"{prefix}_kinds"] = np.array(kinds)
    return out


def decode(g, prefix: str) -> pd.DataFrame:
    cols = {}
    for j, kind in enumerate(g[f"{prefix}_kinds"].tolist()):
        if kind.startswith("category"):
            cols[j] = pd.Categorical.from_codes(g[f"{prefix}_c{j}_codes"], categories=g[f"{prefix}_c{j}_categories"].tolist(),
                                                ordered=kind == "category_ordered")
        elif kind == "object_bool":
            cols[j] = g[f"{prefix}_c{j}"].astype(object)
        else:
            cols[j] = g[f"{prefix}_c{j}"].astype(kind)
    idx = pd.Index(g[f"{prefix}_index"].tolist(), dtype=str(g[f"{prefix}_index_dtype"]))
    df = pd.DataFrame(cols, index=idx)
    df.columns = g[f"{prefix}_columns"].tolist()
    return df


def main():
    sw = load_reference()
    out = {"meta": np.array(f"numpy {np.__version__}; pandas {pd.__version__}; reference squidpy tl.sliding_window")}
    for i, (name, kw) in enumerate(CASES):
        df = sw.sliding_window(make_adata(name), copy=True, **kw)
        out.update(encode(df, f"case{i}"))
        pd.testing.assert_frame_equal(decode(out, f"case{i}"), df, check_exact=True)
    for i, (name, kw) in enumerate(COPY_FALSE):
        adata = make_adata(name)
        assert sw.sliding_window(adata, **kw) is None
        out.update(encode(adata.obs, f"inplace{i}"))
        pd.testing.assert_frame_equal(decode(out, f"inplace{i}"), adata.obs, check_exact=True)
    for i, args in enumerate(CORNERS):
        w = sw._calculate_window_corners(*args)
        out.update(encode(w, f"corners{i}"))
        pd.testing.assert_frame_equal(decode(out, f"corners{i}"), w, check_exact=True)
    types_, msgs = [], []
    for name, kw in ERRORS:
        try:
            sw.sliding_window(make_adata(name), copy=True, **kw)
            types_.append(""), msgs.append("")
        except Exception as e:  # noqa: BLE001
            types_.append(type(e).__name__), msgs.append(str(e))
    out["error_types"], out["error_messages"] = np.array(types_), np.array(msgs)
    np.savez_compressed(os.path.join(OUT, "sliding_window.npz"), **out)
    print("wrote sliding_window.npz:", len(CASES), "frames,", len(COPY_FALSE), "written back,", len(CORNERS), "corner frames; errors", list(zip(types_, msgs)))


if __name__ == "__main__":
    main()
