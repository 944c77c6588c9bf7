"""GPU parity of the region replay (shuffle_algo 9) split at its last full round.  When a chunk's permutations leave the
persistent grid's last round partial, that round runs as a second launch while the label groups of the whole rounds are
transposed beside it.  The counts must equal the list replay's (algo 7) or the oracle's: with the split (the split point not
a multiple of 64), with a whole number of rounds and with fewer permutations than one round (one launch), with library
segments (the transpose's row scatter), over two permutation chunks that split each, and with the overlap switched off."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

import squidpy_b200 as sq
from oracle import ref
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import NhoodPlan
from tools import synth

pytestmark = pytest.mark.gpu


def _counts(g, n_cls, base, st, algo, lib=None, n_libs=0, **opts):
    plan = NhoodPlan(g.indptr, g.indices, n_cls)
    plan.set_option("shuffle_algo", algo)
    plan.set_option("shuffle_threads", 512 if algo == 9 else 1024)
    plan.set_option("shuffle_r", 2)
    for k, v in opts.items():
        plan.set_option(k, v)
    if lib is None:
        plan.set_base(base)
    else:
        plan.set_base(base, lib, n_libs)
    out = plan.permute(st)
    plan.close()
    return out


@pytest.fixture(scope="module")
def hex1m():
    g = synth.hex_graph(1000, 1000)
    base = synth.categorical_labels(g.shape[0], 30, seed=0).cat.codes.to_numpy().astype(np.uint32)
    return g, base


def _grid():
    return 2 * sq.default_context(0).sm_count  # two 512-thread replay CTAs per SM at 1M u8 spots


@pytest.mark.parametrize("case", ["split", "whole_rounds", "below_one_round"])
def test_full_size_equals_list_replay(hex1m, case):
    """configs[1] shape: grid + 70 permutations split after one round (4 whole groups of 64 at 132 SMs, the fifth group
    straddles the split); 2 x grid and grid - 40 run one launch."""
    g, base = hex1m
    grid = _grid()
    P = {"split": grid + 70, "whole_rounds": 2 * grid, "below_one_round": grid - 40}[case]
    st = spawn_states(21, P)
    got = _counts(g, 30, base, st, 9)
    np.testing.assert_array_equal(got, _counts(g, 30, base, st, 7))
    if case == "split":
        np.testing.assert_array_equal(_counts(g, 30, base, st, 9, tail_overlap=0), got)


def test_full_size_library_segments(hex1m):
    """Three interleaved libraries: the label rows are in library-grouped order and the transpose scatters them back."""
    g, base = hex1m
    lib = np.random.default_rng(4).integers(0, 3, g.shape[0]).astype(np.int32)
    st = spawn_states(22, _grid() + 70)
    got = _counts(g, 30, base, st, 9, lib, 3)
    np.testing.assert_array_equal(got, _counts(g, 30, base, st, 7, lib, 3))


def test_full_size_two_chunks(hex1m):
    """perm_chunk 320: chunks of 320 and 300 permutations, each past one round of the grid and split again."""
    g, base = hex1m
    st = spawn_states(23, 620)
    got = _counts(g, 30, base, st, 9, perm_chunk=320)
    np.testing.assert_array_equal(got, _counts(g, 30, base, st, 7, perm_chunk=320))


@pytest.mark.parametrize("n_cls", [30, 300])
def test_small_grid_equals_oracle(n_cls):
    """A 100-CTA grid on a 3000-node chain in two library segments, u8 and u16 labels: 170 permutations split at 100 (one
    group under the last round), 200 and 90 do not split, and 460 in chunks of 256 and 204 split in both."""
    n = 3000
    g = sp.csr_matrix((np.ones(n - 1, np.float32), (np.arange(n - 1), np.arange(1, n))), shape=(n, n))
    base = (np.arange(n) * 13 % n_cls).astype(np.uint32)
    lib = (np.arange(n) * 7 % 2).astype(np.int32)
    for P, chunk in ((170, 0), (200, 0), (90, 0), (460, 256)):
        st = spawn_states(24 + P, P)
        got = _counts(g, n_cls, base, st, 9, lib, 2, shuffle_ctas=100, perm_chunk=chunk)
        np.testing.assert_array_equal(got, ref.nhood_perm_counts(g.indptr, g.indices, base, n_cls, st, lib, 2))
