"""Generate tests/golden/delaunay.npz: the UNMODIFIED reference DelaunayBuilder (loaded through oracle/_refload.py) on inputs
whose triangulation is unique, with every post-processing option, float32 / int64 coordinates, interval bounds between float32
neighbours, an interleaved two-library case and the error cases (the reference's spectral transform is numba code that does not
run here; the project's spectral path is pinned by the other graph goldens); plus, for exactly and nearly cocircular inputs and duplicates,
the exact restatement's graph (tests/delaunay_ref.py) beside scipy's.  Run from the repository root:
``python tests/golden/make_golden_delaunay.py``."""

from __future__ import annotations

import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden", "delaunay.npz")


def _f32_between(d):
    """Bounds that cast to float32 values of the data but lie strictly between float32 neighbours in float64."""
    d = np.unique(d[d > 0])
    lo32, hi32 = d[len(d) // 5], d[4 * len(d) // 5]
    ulp_lo = float(np.spacing(np.float32(lo32)))
    ulp_hi = float(np.spacing(np.float32(hi32)))
    return (float(lo32) + 0.25 * ulp_lo, float(hi32) - 0.25 * ulp_hi)


def unique_inputs():
    from tools import synth

    rng = np.random.default_rng(0)
    k = 300
    t = np.arange(k) * (2 * np.pi / k)
    return {
        "uniform": rng.uniform(0, 1000, (700, 2)),
        "clustered": synth.thomas_points(700, n_parents=8, sigma=30.0, extent=1500.0, seed=2),
        "hex": synth.hex_coords(20, 20) + np.random.default_rng(3).uniform(-1e-3, 1e-3, (400, 2)),
        "wheel": np.vstack([[0.0, 0.0], np.c_[np.cos(t), np.sin(t)] * 100.0]),
        "small": np.random.default_rng(5).uniform(0, 10, (150, 2)),
    }


OPTIONS = [dict(), dict(radius=60.0), dict(radius=(80.0, 20.0)), dict(percentile=90.0), dict(radius=30.0, transform="cosine"),
           dict(transform="cosine", set_diag=True), dict(radius=50.0, percentile=50.0, set_diag=True)]


def cocircular_inputs():
    base = np.array([(5, 0), (4, 3), (3, 4), (0, 5), (-3, 4), (-4, 3), (-5, 0), (-4, -3), (-3, -4), (0, -5), (3, -4), (4, -3)], float)
    lat = np.stack(np.meshgrid(np.arange(12), np.arange(12)), -1).reshape(-1, 2).astype(float)
    lat = lat[np.random.default_rng(4).permutation(lat.shape[0])]
    near = np.stack(np.meshgrid(np.arange(10), np.arange(10)), -1).reshape(-1, 2) * 0.1
    base_u = np.stack(np.meshgrid(np.arange(10), np.arange(10)), -1).reshape(-1, 2).astype(float) * 0.1 + 1000.0
    steps = np.random.default_rng(6).integers(-1, 2, base_u.shape)
    ulp = np.where(steps > 0, np.nextafter(base_u, np.inf), np.where(steps < 0, np.nextafter(base_u, -np.inf), base_u))
    rng = np.random.default_rng(7)
    pts = rng.uniform(0, 100, (200, 2))
    dup = np.vstack([pts, pts[rng.integers(0, 200, 50)]])
    dup = dup[rng.permutation(dup.shape[0])]
    return {
        "lattice": (lat, "exact"),
        "circles": (np.vstack([base + off for off in [(0, 0), (20, 0), (0, 20), (20, 20)]]), "exact"),
        "lattice_0.1": (near, "near"),
        "lattice_ulp": (ulp, "near"),
        "duplicates": (dup, "dup"),
    }


def main() -> None:
    import scipy.sparse as sp

    from oracle import _refload
    from tests.delaunay_ref import delaunay_rows

    nb = _refload.load()["nb"]
    out: dict[str, np.ndarray] = {}
    meta: dict[str, object] = {"cases": [], "errors": [], "cocircular": []}

    def put(key, adj, dst):
        for name, m in (("adj", adj), ("dst", dst)):
            m = sp.csr_matrix(m)
            m.sort_indices()
            out[f"{key}|{name}|indptr"] = m.indptr.astype(np.int64)
            out[f"{key}|{name}|indices"] = m.indices.astype(np.int32)
            out[f"{key}|{name}|data"] = m.data

    def case(name, xy, opt):
        key = f"{name}|{json.dumps(opt, sort_keys=True)}"
        put(key, *nb.DelaunayBuilder(**opt).build(xy))
        meta["cases"].append({"key": key, "coords": name, "opt": opt})

    for name, xy in unique_inputs().items():
        out[f"coords|{name}"] = xy
        for opt in OPTIONS:
            case(name, xy, opt)
    xy32 = np.random.default_rng(8).uniform(0, 1000, (600, 2)).astype(np.float32)
    out["coords|f32"] = xy32
    d = nb.DelaunayBuilder().build(xy32)[1].data
    lo, hi = _f32_between(d)
    for opt in [dict(), dict(radius=(lo, hi)), dict(radius=hi), dict(percentile=33.3), dict(percentile=90.0, radius=(lo, 1e9)),
                dict(transform="cosine", radius=hi)]:
        case("f32", xy32, opt)
    xi = np.unique(np.random.default_rng(9).integers(0, 400, (500, 2)), axis=0).astype(np.int64)
    out["coords|i64"] = xi
    for opt in [dict(), dict(radius=(5.0, 30.0)), dict(percentile=50.0, set_diag=True)]:
        case("i64", xi, opt)
    # two interleaved libraries, built per library and combined as the reference's _run does
    xl = np.random.default_rng(10).uniform(0, 500, (800, 2))
    codes = np.random.default_rng(11).integers(0, 2, 800)
    out["coords|lib"], out["codes|lib"] = xl, codes
    for opt in [dict(), dict(radius=40.0, set_diag=True)]:
        b = nb.DelaunayBuilder(**opt)
        mats, ixs = [], []
        for code in range(2):
            idx = np.where(codes == code)[0]
            mats.append(b.build(xl[idx]))
            ixs.extend(idx.tolist())
        key = f"lib|{json.dumps(opt, sort_keys=True)}"
        put(key, *b.combine(mats, ixs))
        meta["cases"].append({"key": key, "coords": "lib", "opt": opt, "library": True})
    errs = {"two": np.array([[0.0, 0.0], [1.0, 1.0]]), "collinear": np.array([[0.0, 0.0], [1.0, 1.0], [2.0, 2.0], [3.0, 3.0]]),
            "dup_collinear": np.array([[0.0, 0.0], [0.0, 0.0], [1.0, 1.0], [1.0, 1.0]]), "nan": np.array([[0.0, 0.0], [1.0, np.nan], [2.0, 1.0]])}
    for name, xy in errs.items():
        out[f"coords|err_{name}"] = xy
        try:
            nb.DelaunayBuilder().build(xy)
            raise AssertionError(name)
        except Exception as e:  # noqa: BLE001 - the type and message are the golden
            meta["errors"].append({"coords": f"err_{name}", "type": type(e).__name__, "message": str(e).splitlines()[0]})
    from scipy.spatial import Delaunay

    for name, (xy, kind) in cocircular_inputs().items():
        out[f"coords|{name}"] = xy
        ip, ix = delaunay_rows(xy)
        out[f"exact|{name}|indptr"], out[f"exact|{name}|indices"] = ip, ix
        rp, rx = Delaunay(xy).vertex_neighbor_vertices
        m = sp.csr_matrix((np.ones(rx.size), rx, rp), shape=(xy.shape[0],) * 2)
        m.sort_indices()
        out[f"qhull|{name}|indptr"], out[f"qhull|{name}|indices"] = m.indptr.astype(np.int64), m.indices.astype(np.int32)
        meta["cocircular"].append({"coords": name, "kind": kind})
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(meta['cases'])} cases, {len(meta['errors'])} errors, {len(meta['cocircular'])} restated inputs")


if __name__ == "__main__":
    main()
