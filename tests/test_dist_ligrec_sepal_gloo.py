"""ligrec and sepal under torch.distributed (gloo, world sizes 2 and 3): the sharding and the single collective per call.

The device calls are replaced by their numpy restatements (``oracle.ref.ligrec_counts`` behind the five library entry points
ligrec's permutation test uses; a column scorer for sepal), so the host logic runs without a GPU:
  * the ranks' permutation ranges partition ``[0, n_perms)``, a rank without permutations makes no library call, and the
    reduced counts equal the single-process counts (also at ``n_perms=1``, and for ``seed=None`` the ranks agree);
  * sepal's ranks score disjoint gene ranges and every rank returns the frame one process computes alone, also with
    ``use_raw=True`` when every worker hashes strings with its own ``PYTHONHASHSEED``."""

from __future__ import annotations

import os
import socket
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Every worker first re-executes itself with a hash seed of its own: the order of a set of strings then differs between the
# ranks, as it does between torchrun workers that inherit no PYTHONHASHSEED.
RESEED = textwrap.dedent(
    """
    import os, sys
    _want = str(101 + 37 * int(os.environ["RANK"]))
    if os.environ.get("PYTHONHASHSEED") != _want:
        os.execve(sys.executable, [sys.executable] + sys.argv, dict(os.environ, PYTHONHASHSEED=_want))
    sys.path.insert(0, os.environ["SQB_ROOT"])
    """
)

WORKER = RESEED + textwrap.dedent(
    """
    import ctypes as C
    import threading
    from datetime import timedelta

    import numpy as np
    import pandas as pd
    import scipy.sparse as sp
    import torch.distributed as dist

    import squidpy_b200 as sq
    from oracle import ref
    from squidpy_b200._dist import world
    from squidpy_b200.gr import _ligrec, _sepal
    from tools import synth


    class FakeCtx:
        device = 0
        handle = None
        lock = threading.RLock()


    def arr(ptr, ctype, shape):
        return np.ctypeslib.as_array((ctype * int(np.prod(shape))).from_address(ptr)).reshape(shape)


    class FakeLib:
        \"\"\"The library entry points of ligrec's permutation test, counting with oracle.ref.ligrec_counts.\"\"\"

        def __init__(self):
            self.calls, self.uploads = 0, []

        def sqb_nhood_create(self, ctx, n, nnz, indptr, indices, n_cls, out):
            self.calls += 1
            self.n, self.n_cls = n, n_cls
            return 0

        def sqb_nhood_set_base(self, h, lab, lib_codes, n_libs):
            self.calls += 1
            self.lab = arr(lab, C.c_uint32, (self.n,)).copy()
            return 0

        def sqb_nhood_permute_upload(self, h, states, n):
            self.calls += 1
            assert n >= 1
            self.states = arr(states, C.c_uint64, (n, 6)).copy()
            self.uploads.append(self.states)
            return 0

        def sqb_ligrec_counts(self, h, data, n_genes, inv, mean, inter, n_inter, cp, n_cp, valid, out):
            self.calls += 1
            got = ref.ligrec_counts(arr(data, C.c_double, (self.n, n_genes)), self.lab, self.n_cls, self.states,
                                    arr(inv, C.c_double, (self.n_cls,)), arr(mean, C.c_double, (self.n_cls, n_genes)),
                                    arr(inter, C.c_int32, (n_inter, 2)), arr(cp, C.c_int32, (n_cp, 2)),
                                    arr(valid, C.c_uint8, (n_inter, n_cp)).astype(bool))
            arr(out, C.c_int64, (n_inter, n_cp))[:] = got
            return 0

        def sqb_nhood_destroy(self, h):
            self.calls += 1


    def column_score(vals, sat, sat_idx, unsat, unsat_idx, **kw):
        \"\"\"Stands in for sepal's diffusion: one float64 per column, a function of that column alone.\"\"\"
        scored.append(vals.shape[1])
        dense = vals.toarray() if sp.issparse(vals) else np.asarray(vals)
        return dense.sum(axis=0, dtype=np.float64) + 0.125 * (dense > 1).sum(axis=0)


    fake, scored = FakeLib(), []
    _ligrec.load = lambda: fake
    _ligrec.default_context = _sepal.default_context = lambda device=None: FakeCtx()
    _sepal.sepal_idxs = lambda conn, spatial, max_neighs, device=None: _sepal._host_idxs(conn, spatial, max_neighs)
    _sepal.sepal_scores = column_score

    # ---- inputs
    rng = np.random.default_rng(0)
    n = 240
    genes = [f"g{i:02d}" for i in range(20)]
    x = rng.poisson(0.9, (n, len(genes))).astype(np.float64) * rng.random((n, len(genes))) * 3
    obs = pd.DataFrame({"cl": pd.Categorical(rng.choice(["a", "b", "c", "d"], n))}, index=[f"c{i}" for i in range(n)])
    inter = pd.DataFrame({"source": [genes[i] for i in rng.integers(0, 20, 25)], "target": [genes[i] for i in rng.integers(0, 20, 25)]})
    lig_ad = sq.AnnDataLite(X=x, obs=obs, var=pd.DataFrame(index=genes))
    lig_kw = dict(interactions=inter, copy=True, use_raw=False, threshold=0.05)
    PERMS = (1, 2, 23, 40)

    g, co = synth.hex_graph(12, 13), synth.hex_coords(12, 13)
    m = g.shape[0]
    sx = rng.poisson(1.2, (m, 30)).astype(np.float64)
    sx[:, 7] = sx[:, 3]  # equal scores: the order of ties follows the gene list
    sx[:, 21] = sx[:, 3]
    raw_names = [f"r{i:02d}" for i in range(30)]
    raw = sq.AnnDataLite(X=sp.csr_matrix(sx), obs=pd.DataFrame(index=[f"s{i}" for i in range(m)]), var=pd.DataFrame(index=raw_names))
    sep_ad = sq.AnnDataLite(X=sx[:, :20], obsp={"spatial_connectivities": g}, obsm={"spatial": co}, var=pd.DataFrame(index=raw_names[:20]),
                            raw=raw)
    SEPAL = {"host": dict(), "one_gene": dict(genes="r05"), "raw": dict(use_raw=True, genes=raw_names[::-1] + ["zz"])}

    # ---- every call in one process first (before the process group exists)
    alone_lig = {p: sq.gr.ligrec(lig_ad, "cl", n_perms=p, seed=11, **lig_kw) for p in PERMS}
    alone_sep = {k: sq.gr.sepal(sep_ad, 6, copy=True, **kw) for k, kw in SEPAL.items()}
    df = pd.DataFrame(x, columns=list(range(20)))
    df["clusters"] = pd.Categorical(rng.integers(0, 4, n), categories=[0, 1, 2, 3])
    cpairs = np.array([(a, b) for a in range(4) for b in range(4)])
    inter_pos = rng.integers(0, 20, (30, 2))
    alone_counts = _ligrec.ligrec_analysis(df, inter_pos, cpairs, threshold=0.05, n_perms=23, seed=4, ctx=FakeCtx())

    dist.init_process_group("gloo", timeout=timedelta(seconds=120))
    rank, ws = world()
    assert ws == int(os.environ["WORLD_SIZE"]) and ws > 1

    # ---- ligrec: permutations partitioned, counts reduced
    full_index = {}
    for p in PERMS:
        full_index[p] = {ref.spawn_states(11, p)[i].tobytes(): i for i in range(p)}
        fake.calls, fake.uploads = 0, []
        got = sq.gr.ligrec(lig_ad, "cl", n_perms=p, seed=11, **lig_kw)
        mine = [full_index[p][row.tobytes()] for up in fake.uploads for row in up]
        shards = [None] * ws
        dist.all_gather_object(shards, mine)
        flat = sorted(i for s in shards for i in s)
        assert flat == list(range(p)), f"permutation shards {shards} do not partition [0, {p})"
        assert all(s == list(range(s[0], s[0] + len(s))) for s in shards if s), f"shards are not contiguous: {shards}"
        if not mine:
            assert fake.calls == 0, "a rank without permutations called the library"
        for key in ("means", "pvalues", "metadata"):
            assert got[key].equals(alone_lig[p][key]), f"ligrec {key} at n_perms={p} differs from one process"

    res = _ligrec.ligrec_analysis(df, inter_pos, cpairs, threshold=0.05, n_perms=23, seed=4, ctx=FakeCtx())
    assert res.pvalues.tobytes() == alone_counts.pvalues.tobytes() and res.means.tobytes() == alone_counts.means.tobytes()
    valid = ~np.isnan(res.pvalues)
    grp = df.groupby("clusters", observed=True)
    exp = ref.ligrec_counts(x, df["clusters"].cat.codes.to_numpy(), 4, ref.spawn_states(4, 23), 1.0 / grp.size().to_numpy().astype(float),
                            grp.mean().to_numpy(), inter_pos.astype(np.int32), cpairs.astype(np.int32), valid)
    assert (np.where(valid, res.pvalues, 0.0) == exp / 23).all(), "reduced counts differ from the one-process counts"
    # seed=None: one entropy draw for all ranks, so the ranks agree
    unseeded = _ligrec.ligrec_analysis(df, inter_pos, cpairs, threshold=0.05, n_perms=23, seed=None, ctx=FakeCtx()).pvalues
    every = [None] * ws
    dist.all_gather_object(every, unseeded.tobytes())
    assert len(set(every)) == 1, "ranks returned different p-values for seed=None"

    # ---- sepal: genes sharded, frames gathered in gene order
    local_raw = list(set(raw_names) & set(raw_names[::-1] + ["zz"]))
    orders = [None] * ws
    dist.all_gather_object(orders, local_raw)
    assert any(o != orders[0] for o in orders), "the ranks' hash seeds give one set order: the use_raw case tests nothing"
    for k, kw in SEPAL.items():
        scored.clear()
        got = sq.gr.sepal(sep_ad, 6, copy=True, **kw)
        frames = [None] * ws
        dist.all_gather_object(frames, (got, sum(scored)))
        n_genes = len(got)
        assert sum(f[1] for f in frames) == n_genes, f"sepal {k}: the ranks scored {[f[1] for f in frames]} of {n_genes} genes"
        assert all(f[0].equals(got) and list(f[0].index) == list(got.index) for f in frames), f"sepal {k}: ranks differ"
        if rank == 0:  # rank 0's gene list is the one every rank shards: the frame rank 0 computes alone
            assert got.equals(alone_sep[k]) and list(got.index) == list(alone_sep[k].index), f"sepal {k} differs from one process"
        for name, val in got["sepal_score"].items():
            col = sx[:, raw_names.index(name)]
            assert val == col.sum() + 0.125 * (col > 1).sum(), f"sepal {k}: gene {name} carries another gene's score"
    dist.destroy_process_group()
    print("RANK_OK", rank)
    """
)


def free_port() -> int:
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def launch(script: str, tmp_path, nproc: int, timeout: int, args=(), **env) -> subprocess.CompletedProcess:
    """``torch.distributed.run`` with ``nproc`` local workers on a free port, ``script tmp_path *args`` each; returns after every
    worker has exited (on a timeout the launcher is terminated, and it stops its workers)."""
    path = tmp_path / "worker.py"
    path.write_text(script)
    env = dict(os.environ, SQB_ROOT=ROOT, PYTHONPATH=ROOT, **env)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), str(path), str(tmp_path), *map(str, args)]
    proc = subprocess.Popen(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    try:
        out, err = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        proc.terminate()
        try:
            out, err = proc.communicate(timeout=60)
        except subprocess.TimeoutExpired:
            proc.kill()
            out, err = proc.communicate()
        err += f"\n[launcher terminated after {timeout} s]"
    return subprocess.CompletedProcess(cmd, proc.returncode, out, err)


@pytest.mark.parametrize("nproc", [2, 3])
def test_ligrec_sepal_sharding_gloo(tmp_path, nproc):
    out = launch(WORKER, tmp_path, nproc, timeout=300)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-6000:]
    assert out.stdout.count("RANK_OK") == nproc, out.stdout
