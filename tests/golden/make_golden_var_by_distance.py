"""Generates tests/golden/var_by_distance.npz: the UNMODIFIED reference ``tl.var_by_distance`` (a squidpy source checkout, ``$SQUIDPY_REF``,
through the stub-import loader ``oracle/_refload.py``) on a fixture that reaches every branch and quirk of its frame assembly.
Only runnable where the reference tree exists; the output is committed.

    python tests/golden/make_golden_var_by_distance.py

Fixture: two slides on an integer lattice (distances tie exactly), clusters ``a`` / ``b`` / ``c`` where slide ``s1`` has no
``c``, one row per slide with a NaN coordinate in ``obsm["spatial"]`` and, in ``obsm["alt"]``, NaN rows elsewhere (the
reference searches ``obsm["spatial"]`` but re-inserts NaN at the rows of ``obsm[spatial_key]``), obs names whose
lexicographic order is not the row order, slides interleaved in row order.  The frames are stored without pickles: column
names, float columns, categorical codes and categories, and the index.  The exception type of every error case is stored
by name.
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

# (groups, kwargs): groups ("arr", [...]) is passed as a 1-D ndarray of those names
CASES = [
    ("a", dict(cluster_key="cluster")),
    ("a", dict(cluster_key="cluster", metric="manhattan")),
    ("a", dict(cluster_key="cluster", library_key="library")),
    ("c", dict(cluster_key="cluster", library_key="library", metric="chebyshev")),
    (["a", "c"], dict(cluster_key="cluster", library_key="library")),
    (["c", "a"], dict(cluster_key="cluster", library_key="library", metric="l1")),
    (("arr", ["a", "b"]), dict(cluster_key="cluster", library_key="library")),
    (("arr", ["c", "a"]), dict(cluster_key="cluster", library_key="library", metric="infinity")),
    (("arr", ["b"]), dict(cluster_key="cluster", library_key="library")),
    (["a", "b"], dict(cluster_key="cluster")),
    (("arr", ["b", "a", "c"]), dict(cluster_key="cluster", metric="cityblock")),
    ("b", dict(cluster_key="cluster", library_key="library", library_id="s1")),
    (["a", "b"], dict(cluster_key="cluster", library_key="library", library_id=["s1", "s0"], metric="minkowski")),
    (["b"], dict(cluster_key="cluster", library_key="library", library_id=["s0"], covariates="cov")),
    (["a", "b"], dict(cluster_key="cluster", library_key="library", covariates=["cov", "kind"])),
    ("a", dict(cluster_key="cluster", covariates=["kind", "cluster"], metric="l2")),
    ([[1.0, 2.0], [7.5, 0.25]], dict(library_key="library")),
    ([[2.0, 3.0], [0.0, 0.0]], dict(library_key="library", library_id=["s1", "s0"], metric="p")),
    ([[1.5, 2.5]], dict(cluster_key="cluster")),
    ([[4.0, 4.0]], dict(cluster_key="cluster", metric="chebyshev", covariates="cov")),
    ("a", dict(cluster_key="cluster", spatial_key="alt")),
    (["a", "c"], dict(cluster_key="cluster", library_key="library", spatial_key="alt", metric="manhattan")),
    ("b", dict(cluster_key="cluster", library_key="library", design_matrix_key="dm")),
]

# (groups, kwargs) the reference rejects; the stored value is the exception type's name
ERRORS = [
    (("tuple", ["a"]), dict(cluster_key="cluster")),
    (("arr2d", [["a", "b"]]), dict(cluster_key="cluster")),
    ("a", dict(cluster_key="cluster", library_key="library", library_id="s9")),
    ([[1.0, 2.0]], dict(library_key="library")),
    ([[1.0, 2.0], [2.0, 3.0]], dict(cluster_key="cluster")),
    ("a", dict(cluster_key="cluster", metric="haversine")),
    ("a", dict(cluster_key="cluster", metric="nonsense")),
    ("a", dict(cluster_key="cluster", metric="seuclidean")),
    ("z", dict(cluster_key="cluster")),
    ([[1.0, 2.0]], dict()),
    ("a", dict(cluster_key="cluster", library_key=3)),
]


def groups_arg(g):
    if isinstance(g, tuple):
        kind, v = g
        return np.array(v) if kind in ("arr", "arr2d") else tuple(v)
    return g


def fixture():
    """obs (cluster / library categoricals, two covariates), obsm["spatial"] and obsm["alt"]."""
    rng = np.random.default_rng(7)
    gx, gy = np.meshgrid(np.arange(9), np.arange(7))
    s0 = np.stack([gx.ravel(), gy.ravel()], 1)
    gx, gy = np.meshgrid(np.arange(6), np.arange(5))
    s1 = np.stack([gx.ravel() * 2, gy.ravel() * 2 + 1], 1)
    xy = np.concatenate([s0, s1]).astype(np.float64)
    lib = np.repeat([0, 1], [len(s0), len(s1)])
    cl = np.where(lib == 0, rng.integers(0, 3, len(lib)), rng.integers(0, 2, len(lib)))
    perm = rng.permutation(len(lib))
    xy, lib, cl = xy[perm], lib[perm], cl[perm]
    n = len(lib)
    names = [f"cell{int(i)}" for i in rng.permutation(n) * 7 % 1000]
    obs = pd.DataFrame({
        "cluster": pd.Categorical.from_codes(cl, categories=["a", "b", "c"]),
        "library": pd.Categorical.from_codes(lib, categories=["s0", "s1"]),
        "cov": rng.random(n),
        "kind": pd.Categorical.from_codes(rng.integers(0, 2, n), categories=["x", "y"]),
    }, index=pd.Index(names))
    nan0 = [int(np.flatnonzero(lib == 0)[3]), int(np.flatnonzero(lib == 1)[5])]
    nan1 = [int(np.flatnonzero(lib == 0)[10]), int(np.flatnonzero(lib == 1)[1])]
    spatial = xy.copy()
    spatial[nan0[0], 0] = np.nan
    spatial[nan0[1], 1] = np.nan
    alt = xy.copy()
    alt[nan1[0], 1] = np.nan
    alt[nan1[1], :] = np.nan
    return obs, {"spatial": spatial, "alt": alt}


class RowAnnData:
    """The AnnData surface the reference's var_by_distance reads: obs, obsm, obs_names and boolean row indexing."""

    def __init__(self, obs, obsm):
        self.obs = obs
        self.obsm = dict(obsm)

    @property
    def obs_names(self):
        return self.obs.index

    def __getitem__(self, mask):
        m = np.asarray(mask, dtype=bool)
        return RowAnnData(self.obs[m], {k: v[m] for k, v in self.obsm.items()})


def make_adata(cls=None):
    obs, obsm = fixture()
    if cls is None:
        return RowAnnData(obs, obsm)
    return cls(obs=obs, obsm=obsm, shape=(len(obs), 0))


def load_reference():
    from oracle import _refload

    _refload.load()
    m = types.ModuleType("squidpy.tl")
    m.__path__ = [f"{_refload.REF_SRC}/squidpy/tl"]  # type: ignore[attr-defined]
    sys.modules["squidpy.tl"] = m
    return importlib.import_module("squidpy.tl._var_by_distance")


def encode(df: pd.DataFrame, prefix: str) -> dict[str, np.ndarray]:
    """A frame as plain arrays: column names, per column its kind and values (categorical: codes and categories), index."""
    out = {f"{prefix}_columns": np.array([str(c) for c in df.columns]), f"{prefix}_index": np.array([str(i) for i in df.index]),
           f"{prefix}_index_dtype": np.array(str(df.index.dtype))}
    kinds = []
    for j, c in enumerate(df.columns):
        s = df.iloc[:, j]
        if isinstance(s.dtype, pd.CategoricalDtype):
            kinds.append("category")
            out[f"{prefix}_c{j}_codes"] = np.asarray(s.cat.codes, dtype=np.int64)
            out[f"{prefix}_c{j}_categories"] = np.array([str(x) for x in s.cat.categories])
        else:
            kinds.append(str(s.dtype))
            out[f"{prefix}_c{j}"] = s.to_numpy()
    out[f"{prefix}_kinds"] = np.array(kinds)
    return out


def decode(g, prefix: str) -> pd.DataFrame:
    cols = {}
    for j, (name, kind) in enumerate(zip(g[f"{prefix}_columns"].tolist(), g[f"{prefix}_kinds"].tolist())):
        if kind == "category":
            cols[j] = pd.Categorical.from_codes(g[f"{prefix}_c{j}_codes"], categories=g[f"{prefix}_c{j}_categories"].tolist())
        else:
            cols[j] = g[f"{prefix}_c{j}"].astype(kind)
    idx = pd.Index(g[f"{prefix}_index"].tolist(), dtype=str(g[f"{prefix}_index_dtype"]))
    df = pd.DataFrame(cols, index=idx)
    df.columns = g[f"{prefix}_columns"].tolist()
    return df


def main():
    import sklearn

    vbd = load_reference()
    out = {"meta": np.array(f"numpy {np.__version__}; pandas {pd.__version__}; sklearn {sklearn.__version__}; reference squidpy "
                            "tl.var_by_distance")}
    for i, (groups, kw) in enumerate(CASES):
        df = vbd.var_by_distance(make_adata(), groups_arg(groups), copy=True, **kw)
        out.update(encode(df, f"case{i}"))
        assert decode(out, f"case{i}").equals(df), i
        pd.testing.assert_frame_equal(decode(out, f"case{i}"), df, check_exact=True)
    errs = []
    for groups, kw in ERRORS:
        try:
            vbd.var_by_distance(make_adata(), groups_arg(groups), copy=True, **kw)
            errs.append("")
        except Exception as e:  # noqa: BLE001
            errs.append(type(e).__name__)
    out["errors"] = np.array(errs)
    np.savez_compressed(os.path.join(OUT, "var_by_distance.npz"), **out)
    print("wrote var_by_distance.npz:", len(CASES), "frames; errors", errs)


if __name__ == "__main__":
    main()
