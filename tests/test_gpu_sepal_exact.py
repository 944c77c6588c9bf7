"""sepal's stopping iteration, exactly, against a high-precision restatement of the reference's diffusion loop.

The score is ``dt x (first iteration whose entropy change is <= thresh)``: a decision, not a float.  Wherever that decision
is well conditioned — every ``| |dent_i| - thresh |`` up to the stop is far above the floating-point error of the entropy —
any correct float64 implementation takes it the same way, so the kernel must return ``dt * stop`` bit for bit there, and NaN
exactly where the reference does not stop within ``n_iter``.

``diffusion_trajectory`` restates ``_diffusion`` (``_sepal.py``: ``_laplacian_hex`` / ``_laplacian_rect``, ``_entropy`` with
its ``max(p, eps)`` clamp and its ``sum < eps -> 0`` branch) vectorised over genes, in float64 or in ``np.longdouble``.  The
conditioning threshold tau is measured, not guessed: the largest float64 / long-double entropy difference over the golden
trajectories, times 100 for the kernel's other summation order, FMA contraction and entropy form (``log S - sum x log x / S``).

The CPU tests tie the restatement to ``oracle.ref.sepal_score`` (exact), to the long double and to the golden scores of the
unmodified, numba-fastmath reference (within its tolerance), and bound the effect of the entropy clamp the kernel omits.  The
GPU tests cover both sides of the shared-memory rule with both stencils, small lattices with value edges and non-default
``dt`` / ``thresh``, a gene queue longer than the CTA count, the ``n_iter`` edges and a matrix read from GPU memory."""

from __future__ import annotations

import functools
import os
from typing import NamedTuple

import numpy as np
import pytest

from tests.golden.make_golden_sepal import make_case, square_graph

GOLD = dict(np.load(os.path.join(os.path.dirname(__file__), "golden", "sepal.npz"), allow_pickle=False))
EPS = float(np.finfo(np.float64).eps)
DT, THRESH = 0.001, 1e-8
SEPAL_T = 512  # threads per CTA of sepal_kernel (sepal.cu)


class Trajectory(NamedTuple):
    stop: np.ndarray  # per gene: first iteration with |dent| <= thresh, -1 if none within n_iter
    margin: np.ndarray  # per gene: min over iterations 0..stop (all, without a stop) of | |dent_i| - thresh |; NaN dent -> inf
    s_gap: np.ndarray  # per gene: min over the same iterations of |S / eps - 1|, S the positive saturated total
    ent: np.ndarray  # iterations run x genes: the entropy after each iteration, in the run's dtype

    def conditioned(self, tau: float) -> np.ndarray:
        """Genes whose every decision (the stop test and the ``S < eps`` branch) is far from its threshold."""
        return (self.margin > tau) & (self.s_gap > 1e-6)

    def scores(self, dt: float) -> np.ndarray:
        return np.where(self.stop >= 0, dt * self.stop.astype(np.float64), np.nan)


def diffusion_trajectory(vals, use_hex, n_iter, sat, sat_idx, unsat, unsat_idx, dt=DT, thresh=THRESH, dtype=np.float64,
                         clamp=True) -> Trajectory:
    """``_diffusion`` over the spots x genes matrix ``vals`` in ``dtype``.  ``clamp=False`` takes ``log p`` instead of the
    reference's ``log max(p, eps)``, which is what the kernel computes.  Runs until every gene has stopped or ``n_iter``."""
    conc = np.array(vals, dtype=dtype)
    if conc.ndim == 1:
        conc = conc[:, None]
    n_genes, n_sat = conc.shape[1], sat.shape[0]
    dt, thresh, eps = dtype(dt), dtype(thresh), dtype(EPS)
    prev = np.ones(n_genes, dtype)
    stop = np.full(n_genes, -1, np.int64)
    margin = np.full(n_genes, np.inf)
    s_gap = np.full(n_genes, np.inf)
    ents = []
    dcdt = np.zeros_like(conc)
    with np.errstate(all="ignore"):
        for i in range(n_iter):
            nhood = conc[sat_idx].sum(axis=1)
            c = conc[sat]
            d2 = (2.0 * nhood - 12.0 * c) / 3.0 if use_hex else nhood - 4.0 * c
            dcdt[sat] = d2
            conc[sat] += d2 * dt
            conc[unsat] += dcdt[unsat_idx] * dt
            conc[conc < 0] = 0
            x = conc[sat]
            pos = x > 0
            x = np.where(pos, x, 0)
            s = x.sum(axis=0)
            p = x / s
            lp = np.log(np.maximum(p, eps)) if clamp else np.log(p)
            ent = np.where(s < eps, 0, np.where(pos, -lp * p, 0).sum(axis=0)) / n_sat
            d = np.abs(ent - prev)
            run = stop < 0
            gap = np.abs(d - thresh).astype(np.float64)
            margin[run] = np.minimum(margin[run], np.where(np.isnan(gap), np.inf, gap)[run])
            s_gap[run] = np.minimum(s_gap[run], np.abs(s / eps - 1).astype(np.float64)[run])
            stop[run & (d <= thresh)] = i
            ents.append(ent)
            prev = ent
            if (stop >= 0).all():
                break
    return Trajectory(stop, margin, s_gap, np.array(ents))


# ---- lattices and genes ----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def lattice(name: str):
    """(graph, coordinates, max_neighs, (sat, sat_idx, unsat, unsat_idx)) of a named lattice: the golden ones, a 60 x 60 hex,
    and hex / square lattices of 14 464 (113 x 128) and 14 465 (55 x 263) spots on either side of the shared-memory rule."""
    from squidpy_b200.gr._sepal import _compute_idxs
    from tools import synth

    if name in ("hex", "square"):
        g, co, k, _ = make_case(name)
    else:
        kind, rows, cols = name.split("_")
        rows, cols = int(rows), int(cols)
        if kind == "hex":
            g, co, k = synth.hex_graph(rows, cols), synth.hex_coords(rows, cols), 6
        else:
            (g, co), k = square_graph(rows, cols), 4
    return g, co, k, _compute_idxs(g, co, k)


def field_genes(co: np.ndarray, seed: int, n: int) -> np.ndarray:
    """``n`` spots x genes fields of graded roughness: uniform noise, Poisson(0.3) counts, two smooth bumps, bump + noise."""
    rng = np.random.default_rng(seed)
    xy = (co - co.min(0)) / np.ptp(co, axis=0)
    cols = []
    for q in range(n):
        kind = q % 4
        if kind == 0:
            cols.append(rng.random(len(xy)) * (1 + q))
        elif kind == 1:
            cols.append(rng.poisson(0.3, len(xy)).astype(float))
        else:
            bumps = sum(np.exp(-((xy[:, 0] - rng.random()) ** 2 + (xy[:, 1] - rng.random()) ** 2) / (0.005 + 0.02 * rng.random()))
                        for _ in range(2))
            cols.append(bumps + (kind == 3) * rng.random(len(xy)) * 0.3)
    return np.stack(cols, axis=1)


def edge_genes(co: np.ndarray, sat: np.ndarray, seed: int = 0) -> tuple[list[str], np.ndarray]:
    """Value edges, one gene each: all zeros (the ``S < eps`` branch from the start), a constant, a single spike, negative
    entries (clamped by the first step), a spike whose total lies just below / just above eps, a spike on a 1e-30 floor (``p <
    eps`` far from the spike: the entropy clamp), one NaN / +inf / -inf entry in a noise field (they spread to the neighbours and
    drop out of the entropy through ``x > 0``), and magnitudes near 1e300."""
    rng = np.random.default_rng(seed)
    n = co.shape[0]
    mid = int(sat[np.argmin(np.abs(co[sat] - co.mean(0)).sum(1))])  # the saturated node nearest the lattice's centre
    spike = np.zeros(n)
    spike[mid] = 1.0
    noise = rng.random(n)
    genes = {
        "zeros": np.zeros(n),
        "constant": np.full(n, 2.5),
        "spike": spike,
        "negative": rng.random(n) - 0.3,
        "below_eps": spike * (0.5 * EPS),
        "above_eps": spike * (2.0 * EPS),
        "spike_on_1e-30": np.where(spike > 0, 1.0, 1e-30),
        "nan": np.where(np.arange(n) == mid, np.nan, noise),
        "inf": np.where(np.arange(n) == mid, np.inf, noise),
        "-inf": np.where(np.arange(n) == mid, -np.inf, noise),
        "1e300": noise * 1e300,
    }
    return list(genes), np.stack(list(genes.values()), axis=1)


def trajectory(name: str, vals: np.ndarray, n_iter: int, dt=DT, thresh=THRESH, dtype=np.float64, clamp=True) -> Trajectory:
    _, _, k, idx = lattice(name)
    return diffusion_trajectory(vals, k == 6, n_iter, *idx, dt=dt, thresh=thresh, dtype=dtype, clamp=clamp)


# ---- the conditioning threshold --------------------------------------------------------------------------------------------
GOLDEN_LD_ITER = 4000  # long-double iterations per golden case: the measurement of e stays well under a minute


@functools.lru_cache(maxsize=None)
def golden_runs(name: str):
    """float64 and long-double trajectories of a golden case, capped at ``GOLDEN_LD_ITER``."""
    vals = make_case(name)[3]
    return (trajectory(name, vals, GOLDEN_LD_ITER), trajectory(name, vals, GOLDEN_LD_ITER, dtype=np.longdouble))


@functools.lru_cache(maxsize=None)
def float64_error() -> float:
    """e = max |ent64_i - entLD_i| over every iteration of both golden cases (iterations both precisions ran)."""
    e = 0.0
    for name in ("hex", "square"):
        a, b = golden_runs(name)
        m = min(len(a.ent), len(b.ent))
        x, y = a.ent[:m].astype(np.longdouble), b.ent[:m]
        assert np.array_equal(np.isnan(x), np.isnan(y))
        e = max(e, float(np.nanmax(np.abs(x - y))))
    return e


def tau() -> float:
    return 100.0 * float64_error()


def assert_exact(got: np.ndarray, ref: Trajectory, dt: float, both_outcomes: bool = True, min_conditioned: float = 0.95):
    """The kernel's scores equal ``dt * stop`` bit for bit on every conditioned gene (NaN where the reference never stops)."""
    cond = ref.conditioned(tau())
    assert cond.mean() >= min_conditioned, (cond.mean(), ref.margin)
    if both_outcomes:
        assert (ref.stop[cond] >= 0).any() and (ref.stop[cond] < 0).any(), ref.stop
    exp = ref.scores(dt)
    bad = np.flatnonzero(cond & ~((got == exp) | (np.isnan(got) & np.isnan(exp))))
    assert bad.size == 0, f"genes {bad}: got {got[bad]}, expected {exp[bad]} (stops {ref.stop[bad]})"


# ---- CPU: the restatement --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["hex", "square"])
def test_restatement_equals_oracle_on_golden_cases(name):
    """float64 restatement == ``oracle.ref.sepal_score`` (a per-gene numpy loop) on every golden gene, both outcomes present."""
    from oracle import ref

    _, _, k, idx = lattice(name)
    vals = make_case(name)[3]
    got = golden_runs(name)[0].scores(DT)
    exp = np.array([ref.sepal_score(vals[:, q], k == 6, GOLDEN_LD_ITER, *idx) for q in range(vals.shape[1])])
    np.testing.assert_array_equal(got, exp)
    assert np.isnan(exp).any() and np.isfinite(exp).any()


def test_long_double_agrees_and_tau_is_far_below_thresh():
    """The long-double stops equal the float64 stops on every conditioned golden gene; tau = 100 e is far below thresh (so the
    exact comparisons are not vacuous) and still leaves at least 95 % of the golden genes conditioned."""
    e = float64_error()
    assert 0.0 < e < 1e-15, e
    assert tau() < 1e-4 * THRESH
    for name in ("hex", "square"):
        a, b = golden_runs(name)
        cond = a.conditioned(tau()) & b.conditioned(tau())
        assert cond.mean() >= 0.95, (name, a.margin)
        np.testing.assert_array_equal(a.stop[cond], b.stop[cond])
        assert (a.stop[cond] >= 0).any() and (a.stop[cond] < 0).any()


@pytest.mark.parametrize("name", ["hex", "square"])
def test_restatement_matches_fastmath_golden(name):
    """The restatement against the scores of the unmodified reference (numba fastmath) at the tolerance fastmath needs: the
    same NaN pattern at 30 000 and at 300 iterations, every stop within 2 iterations, 80 % equal."""
    vals = make_case(name)[3]
    full = trajectory(name, vals, 30000).scores(DT)
    exp = GOLD[f"{name}_score"]
    assert np.array_equal(np.isnan(full), np.isnan(exp))
    ok = ~np.isnan(exp)
    d_iter = np.abs(full[ok] - exp[ok]) / DT
    assert (d_iter <= 2.5).all(), d_iter
    assert (d_iter < 0.5).mean() >= 0.8
    short = trajectory(name, vals, 300).scores(DT)
    np.testing.assert_array_equal(np.isnan(short), np.isnan(GOLD[f"{name}_score_300"]))


def test_entropy_clamp_cannot_move_a_conditioned_stop():
    """The reference takes ``log max(p, eps)``; the kernel takes ``log p``.  For one entry with ``p < eps`` the two entropy terms
    differ by ``p (log eps - log p)``, at most ``eps / e`` ~ 8.2e-17 (at ``p = eps / e``), so after the division by ``n_sat``
    the entropies differ by at most 8.2e-17 times the clamped fraction of the saturated spots, and an entropy change by twice
    that.  A spike of 1 on a 1e-30 floor keeps ``p < eps`` on nearly every spot for many iterations: with ``dt = 0.01``,
    ``thresh = 1e-6`` the long-double entropies with and without the clamp differ by at most ~4.2e-18, inside that bound and
    far below tau, and both stop at iteration 1556."""
    name, dt, thresh = "hex", 0.01, 1e-6
    _, co, _, (sat, *_) = lattice(name)
    names, vals = edge_genes(co, sat)
    v = vals[:, names.index("spike_on_1e-30")]
    a = trajectory(name, v, 3000, dt=dt, thresh=thresh, dtype=np.longdouble)
    b = trajectory(name, v, 3000, dt=dt, thresh=thresh, dtype=np.longdouble, clamp=False)
    m = min(len(a.ent), len(b.ent))
    diff = float(np.max(np.abs(a.ent[:m] - b.ent[:m])))
    assert 0.0 < diff <= EPS / np.e, diff  # the clamp is hit, and stays inside the bound
    assert 2 * diff < tau()
    assert a.stop[0] > 1 and a.stop[0] == b.stop[0] and a.margin[0] > tau()


# ---- GPU: the exact stopping iteration -------------------------------------------------------------------------------------
def uses_global_scratch(n: int, optin: int) -> bool:
    """The dispatch rule of ``sepal_impl`` (sepal.cu): ``need = 2 * n * sizeof(double); global = need + 1024 > smem_optin``."""
    return 16 * n + 1024 > optin


# lattices on either side of the rule on an H100 (232 448 B of opt-in shared memory per block: n <= 14 464 fits)
BOUNDARY = [("hex_113_128", False), ("hex_55_263", True), ("square_113_128", False), ("square_55_263", True)]
BOUNDARY_ITER = 500  # smooth fields stop at once, noise after a few hundred iterations, Poisson counts later: both outcomes
# (dt, thresh, n_iter): the cap leaves genes that stop and genes that do not on every small lattice
PARAMS = [(0.001, 1e-8, 3000), (0.01, 1e-6, 250), (0.0005, 1e-9, 3000)]


def test_dispatch_rule_boundary_on_h100():
    from tests.device_attrs import H100_SMEM_OPTIN

    assert not uses_global_scratch(14464, H100_SMEM_OPTIN) and uses_global_scratch(14465, H100_SMEM_OPTIN)
    for name, global_scratch in BOUNDARY:
        assert uses_global_scratch(lattice(name)[0].shape[0], H100_SMEM_OPTIN) == global_scratch, name


@functools.lru_cache(maxsize=None)
def boundary_case(name: str):
    vals = field_genes(lattice(name)[1], seed=11, n=4)
    return vals, trajectory(name, vals, BOUNDARY_ITER)


@functools.lru_cache(maxsize=None)
def golden_full(name: str) -> Trajectory:
    return trajectory(name, make_case(name)[3], 30000)


@functools.lru_cache(maxsize=None)
def small_case(name: str, dt: float, thresh: float, n_iter: int):
    """The golden genes (or twelve graded fields on the 60 x 60 hex) followed by the value-edge genes."""
    _, co, _, (sat, *_) = lattice(name)
    names, edges = edge_genes(co, sat)
    fields = make_case(name)[3] if name in ("hex", "square") else field_genes(co, seed=60, n=12)
    vals = np.concatenate([fields, edges], axis=1)
    return names, vals, trajectory(name, vals, n_iter, dt=dt, thresh=thresh)


@pytest.fixture(scope="module")
def optin():
    from tests.device_attrs import smem_optin

    return smem_optin()


def _scores(name, vals, **kw):
    from squidpy_b200.gr import sepal_scores

    _, _, k, idx = lattice(name)
    return sepal_scores(vals, *idx, max_neighs=k, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name,global_scratch", BOUNDARY)
def test_exact_stop_on_both_sides_of_the_shared_memory_rule(optin, name, global_scratch):
    from tests.device_attrs import H100_SMEM_OPTIN

    if optin != H100_SMEM_OPTIN:
        pytest.skip(f"boundary case written for {H100_SMEM_OPTIN} B of opt-in shared memory per block, this device has {optin} B")
    assert uses_global_scratch(lattice(name)[0].shape[0], optin) == global_scratch
    vals, ref = boundary_case(name)
    assert (ref.stop == 1).any()  # a smooth field stops after one step
    assert_exact(_scores(name, vals, n_iter=BOUNDARY_ITER), ref, DT)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hex", "square"])
def test_exact_stop_on_golden_genes_at_full_length(name):
    """The golden genes at the default 30 000 iterations: stops up to ~29 500 dependent iterations, and genes that never stop."""
    ref = golden_full(name)
    assert ref.stop.max() > 20000
    assert_exact(_scores(name, make_case(name)[3]), ref, DT)


@pytest.mark.gpu
@pytest.mark.parametrize("dt,thresh,n_iter", PARAMS)
@pytest.mark.parametrize("name", ["hex", "square", "hex_60_60"])
def test_exact_stop_with_value_edges_and_parameters(name, dt, thresh, n_iter):
    names, vals, ref = small_case(name, dt, thresh, n_iter)
    e = vals.shape[1] - len(names)
    edge = dict(zip(names, ref.stop[e:]))
    assert edge["zeros"] == 1 and edge["below_eps"] == 1 and edge["constant"] == 1  # S < eps -> entropy 0; a constant is at rest
    assert (ref.stop[:e] > 1).any()
    got = _scores(name, vals, n_iter=n_iter, dt=dt, thresh=thresh)
    assert_exact(got, ref, dt)
    assert ref.conditioned(tau())[e:].mean() >= 0.9  # the value edges themselves are checked


@pytest.mark.gpu
def test_gene_queue_longer_than_the_cta_count():
    """1 100 genes on a 440-spot lattice: more than the at most 4 x SM-count CTAs of 512 threads, so CTAs take several genes
    from the queue in turn.  Equal, bit for bit, to batches of 100 genes (fewer than one CTA per SM: one gene per CTA), and a
    sample equals the reference."""
    from tests.device_attrs import sm_count

    name, n_genes, batch, n_iter, dt, thresh = "hex", 1100, 100, 400, 0.01, 1e-6
    assert n_genes > (2048 // SEPAL_T) * sm_count() and batch < sm_count()
    vals = field_genes(lattice(name)[1], seed=5, n=n_genes)
    got = _scores(name, vals, n_iter=n_iter, dt=dt, thresh=thresh)
    np.testing.assert_array_equal(got, _scores(name, vals, n_iter=n_iter, dt=dt, thresh=thresh, batch_genes=batch))
    sample = np.sort(np.random.default_rng(1).choice(n_genes, 96, replace=False))
    assert_exact(got[sample], trajectory(name, vals[:, sample], n_iter, dt=dt, thresh=thresh), dt)


@pytest.mark.gpu
def test_n_iter_edges():
    """For every gene that stops at s: ``n_iter = s + 1`` gives the same score, ``n_iter = s`` gives NaN.  One iteration with
    ``thresh >= |ent_0 - 1|`` stops at 0 (the all-zero gene sits exactly on ``|0 - 1| <= 1``)."""
    name = "hex"
    vals = np.concatenate([make_case(name)[3], np.zeros((lattice(name)[0].shape[0], 1))], axis=1)
    full = _scores(name, vals)
    stops = np.rint(full / DT)
    assert np.isfinite(stops).sum() >= 10
    for q in np.flatnonzero(np.isfinite(stops)):
        s = int(stops[q])
        assert _scores(name, vals[:, [q]], n_iter=s + 1)[0] == full[q], (q, s)
        assert np.isnan(_scores(name, vals[:, [q]], n_iter=s)[0]), (q, s)
    assert (_scores(name, vals, n_iter=1, thresh=1.0, dt=0.25) == 0.0).all()
    assert np.isnan(_scores(name, vals, n_iter=1)).all()


@pytest.mark.gpu
def test_device_matrix_against_the_reference(optin):
    """X in GPU memory (a torch CUDA tensor: ``sqb_dense_gather_device`` then ``sqb_sepal_dense``) against the reference, on a
    global-scratch lattice and with the value-edge genes."""
    torch = pytest.importorskip("torch")
    name = "hex_55_263"
    assert uses_global_scratch(lattice(name)[0].shape[0], optin)
    vals, ref = boundary_case(name)
    assert_exact(_scores(name, torch.as_tensor(vals).cuda(), n_iter=BOUNDARY_ITER), ref, DT)
    dt, thresh, n_iter = PARAMS[0]
    _, vals, ref = small_case("hex", dt, thresh, n_iter)
    assert_exact(_scores("hex", torch.as_tensor(vals).cuda(), n_iter=n_iter, dt=dt, thresh=thresh), ref, dt)
