"""CPU checks of the Delaunay builder: the exact predicates of ``csrc/delaunay_pred.h`` (built for the host with g++) agree in
sign with rational arithmetic on random, near-degenerate and wide-exponent inputs; the symbolic perturbation never returns 0
and is invariant under cyclic rotation; argument handling and ``uns_params``."""

from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess
import tempfile
from fractions import Fraction as F

import numpy as np
import pytest

from squidpy_b200.gr import DelaunayBuilder

HDR = os.path.join(os.path.dirname(__file__), "..", "squidpy_b200", "csrc", "delaunay_pred.h")
SRC = r"""
#include "delaunay_pred.h"
extern "C" int t_orient(const double* a, const double* b, const double* c) { return dpred::orient2d(a, b, c); }
extern "C" int t_incircle(const double* a, const double* b, const double* c, const double* d) { return dpred::incircle(a, b, c, d); }
extern "C" int t_incircle_sos(const double* a, const double* b, const double* c, const double* d, long long ia, long long ib, long long ic,
                              long long id) { return dpred::incircle_sos(a, b, c, d, ia, ib, ic, id); }
"""


@pytest.fixture(scope="module")
def pred():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    d = tempfile.mkdtemp()
    src, so = os.path.join(d, "p.cpp"), os.path.join(d, "p.so")
    with open(src, "w") as f:
        f.write(SRC)
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.dirname(HDR), src, "-o", so], check=True)
    lib = C.CDLL(so)
    P = C.POINTER(C.c_double)
    lib.t_orient.argtypes = [P] * 3
    lib.t_incircle.argtypes = [P] * 4
    lib.t_incircle_sos.argtypes = [P] * 4 + [C.c_longlong] * 4
    yield lib
    shutil.rmtree(d, ignore_errors=True)


def _p(v):
    a = (C.c_double * 2)(float(v[0]), float(v[1]))
    return a


def _sgn(x):
    return (x > 0) - (x < 0)


def orient_q(a, b, c):
    a, b, c = [(F(p[0]), F(p[1])) for p in (a, b, c)]
    return _sgn((a[0] - c[0]) * (b[1] - c[1]) - (a[1] - c[1]) * (b[0] - c[0]))


def incircle_q(a, b, c, d):
    a, b, c, d = [(F(p[0]), F(p[1])) for p in (a, b, c, d)]
    rows = [(p[0] - d[0], p[1] - d[1]) for p in (a, b, c)]
    rows = [(x, y, x * x + y * y) for x, y in rows]
    (a1, a2, a3), (b1, b2, b3), (c1, c2, c3) = rows
    return _sgn(a1 * (b2 * c3 - b3 * c2) - a2 * (b1 * c3 - b3 * c1) + a3 * (b1 * c2 - b2 * c1))


def _inputs(rng, kind, n):
    if kind == "random":
        return rng.uniform(-1, 1, (n, 4, 2))
    if kind == "lattice":  # exactly cocircular / collinear
        return rng.integers(-3, 4, (n, 4, 2)).astype(float)
    if kind == "ulp":  # lattice points moved by single ulps
        base = rng.integers(-3, 4, (n, 4, 2)).astype(float) * 0.1 + 1e3
        steps = rng.integers(-2, 3, (n, 4, 2))
        return np.where(steps > 0, np.nextafter(base, np.inf), np.where(steps < 0, np.nextafter(base, -np.inf), base))
    if kind == "exponent":
        scale = 2.0 ** rng.integers(-90, 90, (n, 1, 1))
        return rng.integers(-3, 4, (n, 4, 2)).astype(float) * scale + rng.uniform(-1, 1, (n, 4, 2)) * scale * 2.0**-40
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["random", "lattice", "ulp", "exponent"])
def test_predicates_match_rationals(pred, kind):
    rng = np.random.default_rng(hash(kind) % 2**32)
    for q in _inputs(rng, kind, 400):
        a, b, c, d = q
        assert pred.t_orient(_p(a), _p(b), _p(c)) == orient_q(a, b, c), q
        assert pred.t_incircle(_p(a), _p(b), _p(c), _p(d)) == incircle_q(a, b, c, d), q


def test_perturbation_is_total_and_rotation_invariant(pred):
    rng = np.random.default_rng(1)
    n_zero = 0
    for q in _inputs(rng, "lattice", 3000):
        a, b, c, d = q
        if orient_q(a, b, c) <= 0 or len({tuple(p) for p in q}) < 4:
            continue
        exact = incircle_q(a, b, c, d)
        ids = rng.permutation(10)[:4]
        s = pred.t_incircle_sos(_p(a), _p(b), _p(c), _p(d), *map(int, ids))
        assert s != 0
        if exact != 0:
            assert s == exact
        else:
            n_zero += 1
        s2 = pred.t_incircle_sos(_p(b), _p(c), _p(a), _p(d), int(ids[1]), int(ids[2]), int(ids[0]), int(ids[3]))
        assert s2 == s
    assert n_zero > 10


def test_arguments_and_uns_params():
    assert DelaunayBuilder().uns_params() == {"coord_type": "generic", "radius": None, "transform": None}
    assert DelaunayBuilder(radius=5).uns_params()["radius"] == [0.0, 5.0]
    assert DelaunayBuilder(radius=(9.0, 2.0))._interval() == (2.0, 9.0)
    assert DelaunayBuilder(radius=(9.0, 2.0)).uns_params()["radius"] == [9.0, 2.0]
    assert DelaunayBuilder(transform="spectral").uns_params()["transform"] == "spectral"
    assert DelaunayBuilder()._interval() is None
    with pytest.raises(ValueError):
        DelaunayBuilder(transform="bogus")


def test_restatement_equals_reference_golden_and_stored_rows():
    """tests/delaunay_ref.py reproduces the reference's graph on an input with a unique triangulation, and the restated rows
    stored for the cocircular inputs."""
    import json

    import scipy.sparse as sp

    from tests.delaunay_ref import delaunay_rows

    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "delaunay.npz"))
    meta = json.loads(str(g["meta"]))
    key = next(c["key"] for c in meta["cases"] if c["coords"] == "small" and not c["opt"])
    ip, ix = delaunay_rows(g["coords|small"])
    ref = sp.csr_matrix((g[f"{key}|adj|data"], g[f"{key}|adj|indices"], g[f"{key}|adj|indptr"]))
    assert np.array_equal(ip, ref.indptr) and np.array_equal(ix, ref.indices)
    ip, ix = delaunay_rows(g["coords|circles"])
    assert np.array_equal(ip, g["exact|circles|indptr"]) and np.array_equal(ix, g["exact|circles|indices"])
