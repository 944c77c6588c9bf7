"""Multi-GPU plumbing: one process per GPU, ``torch.distributed`` (NCCL on GPUs, gloo on CPU for tests).

The hot path shards embarrassingly — permutations for ``nhood_enrichment`` and ``ligrec``, features for
``spatial_autocorr`` and ``sepal``, pair tiles for ``co_occurrence``/``ripley`` — so there is exactly ONE collective per call,
on the final small tensor
(SURVEY.md section 8e).  Chunking follows the reference's own rule for splitting work over workers:
contiguous chunks of ``ceil(n / n_workers)`` (``src/squidpy/_utils.py:225-231``).
"""

from __future__ import annotations

import numpy as np


def world() -> tuple[int, int]:
    """(rank, world_size) of the initialised default process group, (0, 1) otherwise."""
    try:
        import torch.distributed as dist
    except Exception:  # pragma: no cover
        return 0, 1
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_range(n: int, rank: int, world_size: int) -> tuple[int, int]:
    step = -(-n // world_size) if n > 0 else 0
    lo = min(rank * step, n)
    return lo, min(lo + step, n)


def shared_seed(seed):
    """``seed`` itself, or — for ``seed=None`` under ``torch.distributed`` — one 128-bit OS-entropy draw made on rank 0 and
    broadcast, so that every rank spawns the same generator family (with per-rank entropy the ranks' shards would come
    from different families: irreproducible for nhood / autocorr, plainly wrong for the Ripley simulations, whose pair
    tiles are summed across ranks)."""
    rank, ws = world()
    if seed is not None or ws == 1:
        return seed
    import torch
    import torch.distributed as dist

    ent = np.random.SeedSequence().entropy if rank == 0 else 0
    words = np.array([(ent >> (32 * k)) & 0xFFFFFFFF for k in range(4)], dtype=np.int64)
    t = torch.from_numpy(words).to(_device_for_backend())
    dist.broadcast(t, src=0)
    words = t.cpu().numpy()
    return int(sum(int(w) << (32 * k) for k, w in enumerate(words)))


def _device_for_backend():
    import torch
    import torch.distributed as dist

    if dist.get_backend() == "nccl":
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def all_gather_rows(local: np.ndarray, n_total: int) -> np.ndarray:
    """Concatenate per-rank row blocks (block ``r`` = ``shard_range(n_total, r, world)``) on every rank."""
    rank, ws = world()
    if ws == 1:
        return local
    import torch
    import torch.distributed as dist

    step = -(-n_total // ws)
    row_shape = local.shape[1:]
    pad = np.zeros((step,) + row_shape, dtype=local.dtype)
    pad[: local.shape[0]] = local
    dev = _device_for_backend()
    # NCCL has no uint32: move bytes
    t = torch.from_numpy(pad.view(np.uint8).reshape(-1)).to(dev)
    out = torch.empty(ws * t.numel(), dtype=torch.uint8, device=dev)
    dist.all_gather_into_tensor(out, t)
    full = out.cpu().numpy().view(local.dtype).reshape((ws * step,) + row_shape)
    return np.ascontiguousarray(full[:n_total])


def broadcast_from_rank0(obj):
    """Rank 0's ``obj`` (any picklable object) on every rank, in one broadcast; ``obj`` itself without a process group."""
    _, ws = world()
    if ws == 1:
        return obj
    import torch.distributed as dist

    box = [obj]
    dist.broadcast_object_list(box, src=0, device=_device_for_backend())
    return box[0]


def all_reduce_sum(local: np.ndarray) -> np.ndarray:
    """Element-wise sum over ranks (int64 / float64 payloads)."""
    rank, ws = world()
    if ws == 1:
        return local
    import torch
    import torch.distributed as dist

    dev = _device_for_backend()
    t = torch.from_numpy(np.ascontiguousarray(local)).to(dev)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t.cpu().numpy()


def sequential_stats(sums_local: np.ndarray, var_step, n_total: int) -> tuple[np.ndarray, np.ndarray]:
    """Per-bin mean and standard deviation over the rows of all ranks (rank r holds the contiguous block
    ``shard_range(n_total, r, world)``), bit-identical to ``full.mean(axis=0)`` / ``full.std(axis=0)`` of the float64
    concatenation, without gathering the rows:

    * the rows are non-negative integer counts, so every partial sum is an exact float64 integer (< 2^53): the int64
      all-reduce of the per-rank sums IS numpy's sequential sum, ``mean = sum / n_total``;
    * ``sum((x - mean)**2)`` is order dependent: ``var_step(mean, acc_in) -> acc_out`` continues numpy's sequential
      accumulation over this rank's rows, the running value travels rank 0 -> 1 -> ... -> last (one small message per hop)
      and the final value is broadcast."""
    rank, ws = world()
    total = all_reduce_sum(np.ascontiguousarray(sums_local, dtype=np.int64))
    mean = total.astype(np.float64) / n_total
    acc = np.zeros_like(mean)
    if ws == 1:
        acc = var_step(mean, acc)
    else:
        import torch
        import torch.distributed as dist

        dev = _device_for_backend()
        if rank > 0:
            t = torch.empty(acc.shape, dtype=torch.float64, device=dev)
            dist.recv(t, src=rank - 1)
            acc = t.cpu().numpy()
        acc = var_step(mean, acc)
        t = torch.from_numpy(np.ascontiguousarray(acc)).to(dev)
        if rank < ws - 1:
            dist.send(t, dst=rank + 1)
        dist.broadcast(t, src=ws - 1)
        acc = t.cpu().numpy()
    return mean, np.sqrt(acc / n_total)


def nccl_cuda() -> bool:
    """True when the default process group runs NCCL (one process per GPU): collectives take device tensors."""
    try:
        import torch.distributed as dist

        return dist.is_available() and dist.is_initialized() and dist.get_backend() == "nccl"
    except Exception:  # pragma: no cover
        return False


GATHER_LIMIT_BYTES = 2 << 30  # gathered counts larger than this go through the rank-to-rank chain instead


def gathered_stats_device(plan, n_total: int, has_rows: bool) -> tuple[np.ndarray, np.ndarray]:
    """Per-bin mean and standard deviation over the permutation counts of ALL ranks under NCCL, with ONE collective: every rank
    copies its block of counts (device to device) into a buffer padded to ``ceil(n_total / world)`` rows, the blocks are
    all-gathered as device tensors (3.6 MB per rank at 30 clusters x 1000 permutations; the blocks of ``shard_range`` are
    contiguous, so row g of the gathered array is global permutation g), and every rank runs the single-GPU statistics kernel
    over the first ``n_total`` rows -- bit-identical to numpy's ``mean`` / ``std`` over the concatenated float64 counts.
    (The rank-to-rank chain of :func:`sequential_stats_device` moves less data but costs a send/recv per rank.)"""
    import ctypes as C

    import torch
    import torch.distributed as dist

    from ._lib import check

    rank, ws = world()
    dev = torch.device("cuda", plan.ctx.device)
    cc = plan.n_cls * plan.n_cls
    step = -(-n_total // ws)
    stream = torch.cuda.current_stream(dev)
    shared = plan.ctx.stream == stream.cuda_stream  # the library launches on torch's current stream: everything is ordered
    local = torch.zeros((step, cc), dtype=torch.int32, device=dev)
    if has_rows:
        if not shared:
            stream.synchronize()
        plan.counts_dev(local.data_ptr())
        if not shared:
            plan.ctx.sync()
    full = torch.empty((ws * step, cc), dtype=torch.int32, device=dev)
    dist.all_gather_into_tensor(full, local)
    stat = torch.empty((2, cc), dtype=torch.float64, device=dev)
    if not shared:
        stream.synchronize()
    check(plan._lib.sqb_nhood_stats_rows_dev(plan.ctx.handle, C.c_void_p(full.data_ptr()), n_total, plan.n_cls,
                                             C.c_void_p(stat[0].data_ptr()), C.c_void_p(stat[1].data_ptr())))
    if not shared:
        plan.ctx.sync()
    res = stat.cpu().numpy()
    return res[0].reshape(plan.n_cls, plan.n_cls), res[1].reshape(plan.n_cls, plan.n_cls)


def stats_device(plan, n_total: int, has_rows: bool) -> tuple[np.ndarray, np.ndarray]:
    """Multi-GPU statistics under NCCL: gather when the gathered counts are small (the usual case), else the chain."""
    _, ws = world()
    if (-(-n_total // ws)) * ws * plan.n_cls * plan.n_cls * 4 <= GATHER_LIMIT_BYTES:
        return gathered_stats_device(plan, n_total, has_rows)
    return sequential_stats_device(plan, n_total, has_rows)


def sequential_stats_device(plan, n_total: int, has_rows: bool) -> tuple[np.ndarray, np.ndarray]:
    """:func:`sequential_stats` with everything on the device (NCCL): the exact int64 per-bin sums of ``plan``'s permutation
    counts are all-reduced as a device tensor, the mean is formed on the device, the variance accumulation travels rank to
    rank as a device tensor (``sqb_nhood_permute_var_chain_dev``), and one (2, C, C) float64 tensor comes back to the host.
    Bit-identical to numpy's ``mean`` / ``std`` over the concatenated float64 counts (same operations in the same order;
    IEEE division and square root are exact in torch as in numpy)."""
    import torch
    import torch.distributed as dist

    rank, ws = world()
    dev = torch.device("cuda", plan.ctx.device)
    cc = plan.n_cls * plan.n_cls
    stream = torch.cuda.current_stream(dev)
    shared = plan.ctx.stream == stream.cuda_stream  # the library launches on torch's current stream: everything is ordered
    sums = torch.zeros(cc, dtype=torch.int64, device=dev)
    if has_rows:
        if not shared:
            stream.synchronize()
        plan.sums_dev(sums.data_ptr())
        if not shared:
            plan.ctx.sync()
    dist.all_reduce(sums, op=dist.ReduceOp.SUM)
    mean = sums.to(torch.float64) / float(n_total)
    acc = torch.zeros(cc, dtype=torch.float64, device=dev)
    if rank > 0:
        dist.recv(acc, src=rank - 1)
    if has_rows:
        out = torch.empty_like(acc)
        if not shared:
            stream.synchronize()
        plan.var_chain_dev(mean.data_ptr(), acc.data_ptr(), out.data_ptr())
        if not shared:
            plan.ctx.sync()
        acc = out
    if rank < ws - 1:
        dist.send(acc, dst=rank + 1)
    dist.broadcast(acc, src=ws - 1)
    res = torch.stack([mean, torch.sqrt(acc / float(n_total))]).cpu().numpy()
    return res[0].reshape(plan.n_cls, plan.n_cls), res[1].reshape(plan.n_cls, plan.n_cls)
