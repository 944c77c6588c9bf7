"""ligrec and sepal on 2 and 3 ranks of a gloo process group sharing one GPU: every rank returns the same frames (order
included), equal bit for bit to the frames of the same calls in one process, and the ranks' logged shards partition the
permutations and the genes -- with an uneven split (1000 permutations on 3 ranks, 23 genes) and ranks left without work
(fewer permutations or genes than ranks).  Each worker hashes strings with its own ``PYTHONHASHSEED``, so sepal's
``use_raw=True`` gene list comes out of its set intersection in a different order on every rank."""

from __future__ import annotations

import pickle

import pytest

from tests.test_dist_ligrec_sepal_gloo import RESEED, launch

pytestmark = pytest.mark.gpu

WORKER = RESEED + """
import logging
import pickle
from datetime import timedelta

import torch.distributed as dist

dist.init_process_group("gloo", timeout=timedelta(seconds=300))
rank = dist.get_rank()


class Shards(logging.Handler):
    def __init__(self):
        super().__init__(logging.INFO)
        self.ranges = []

    def emit(self, record):
        if "(rank %d/%d," in str(record.msg):
            self.ranges.append(tuple(record.args[-4:]))


shards = Shards()
log = logging.getLogger("squidpy_b200")
log.setLevel(logging.INFO)
log.addHandler(shards)

from tests.dist_ligrec_sepal_cases import run

frames = run([int(p) for p in sys.argv[2].split(",")])
with open(os.path.join(sys.argv[1], f"rank{rank}.pkl"), "wb") as f:
    pickle.dump((frames, shards.ranges), f)
dist.destroy_process_group()
print("RANK_OK", rank)
"""


@pytest.mark.parametrize("nproc,perms", [(2, (1, 1000)), (3, (2, 1000))])
def test_ranks_return_the_single_process_frames(tmp_path, nproc, perms):
    from tests.dist_ligrec_sepal_cases import run

    out = launch(WORKER, tmp_path, nproc, timeout=900, args=[",".join(map(str, perms))], SQB_DEVICE="0")
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-6000:]
    assert out.stdout.count("RANK_OK") == nproc, out.stdout
    ranks = []
    for r in range(nproc):
        with open(tmp_path / f"rank{r}.pkl", "rb") as f:
            ranks.append(pickle.load(f))

    # the logged (rank, world, lo, hi) of every call: the ranks' ranges of each call tile [0, n) in rank order
    calls = [rng for _, rng in ranks]
    assert len({len(c) for c in calls}) == 1 and calls[0]
    for k in range(len(calls[0])):
        shard = [c[k] for c in calls]
        assert [s[:2] for s in shard] == [(r, nproc) for r in range(nproc)]
        assert shard[0][2] == 0 and all(a[3] == b[2] for a, b in zip(shard, shard[1:])), shard
    assert any(s[2] == s[3] for c in calls for s in c), "no call left a rank without work"

    frames = [f for f, _ in ranks]
    for name, df in frames[0].items():
        for r in range(1, nproc):
            assert frames[r][name].equals(df) and list(frames[r][name].index) == list(df.index), f"{name}: rank {r} differs from rank 0"

    alone = run(perms)
    assert set(alone) == set(frames[0])
    for name, df in alone.items():
        # sort_index: the use_raw gene list follows this process's string hashing (ties may sort differently)
        assert frames[0][name].sort_index().equals(df.sort_index()), f"{name} differs from the single-process frame"
