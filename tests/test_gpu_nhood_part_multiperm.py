"""GPU parity of the partitioned target generation when every generator warp runs several permutations in turn (more
permutations than the launch has generator warps), so that its two block buffers carry on from one permutation and one
library segment to the next."""

from __future__ import annotations

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import ref
from squidpy_b200._rng import spawn_states
from squidpy_b200.gr import NhoodPlan

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("jgen_threads", [32, 128])
@pytest.mark.parametrize("region", [0, 160])
def test_partitioned_equals_list_replay_many_permutations_per_warp(jgen_threads, region):
    """2500 permutations (an H100 launch makes at most about 1100 generator warps); segments of 2100 and 900 elements take 2
    and 1 blocks, so the blocks of a segment and of a permutation start in either buffer; region 160 gives 14 regions."""
    n, n_cls, P = 3000, 30, 2500
    g = sp.csr_matrix((np.ones(n - 1, np.float32), (np.arange(n - 1), np.arange(1, n))), shape=(n, n))
    base = (np.arange(n) * 13 % n_cls).astype(np.uint32)
    lib = np.zeros(n, np.int32)
    lib[2100:] = 1
    st = spawn_states(11 + region, P)
    out = {}
    for algo in (7, 9):
        plan = NhoodPlan(g.indptr, g.indices, n_cls)
        plan.set_option("shuffle_algo", algo)
        plan.set_option("shuffle_threads", 1024)
        plan.set_option("shuffle_r", 2)
        plan.set_option("shuffle_region", region)
        plan.set_option("jgen_threads", jgen_threads)
        plan.set_base(base, lib, 2)
        out[algo] = plan.permute(st)
        if algo == 9:
            plan.upload(st)
            np.testing.assert_array_equal(plan.shuffled_labels(P - 3, P), ref.shuffle_labels(base, st[P - 3 :], lib, 2))
        plan.close()
    np.testing.assert_array_equal(out[9], out[7])
