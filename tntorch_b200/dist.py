"""Batch sharding across the GPUs of one box (one process per GPU, torch.distributed).

The path shards over independent tensors: rank g decomposes the contiguous slice of the batch it
owns with no data-path collective; ONE all-gather at the end gives every rank all factor cores
(BASELINE.json north_star; SURVEY.md §8e).  Works on any backend (NCCL on the GPUs, gloo in the
CPU test-suite, where only the plumbing is exercised).
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.distributed as dist


def shard_range(batch: int, world: int, rank: int):
    """Contiguous chunk [lo, hi) of a batch of `batch` problems owned by `rank` (ragged tail spread evenly)."""
    base, rem = divmod(batch, world)
    lo = rank * base + min(rank, rem)
    hi = lo + base + (1 if rank < rem else 0)
    return lo, hi


def _dtype_name(dt):
    return str(dt).replace("torch.", "")


def all_gather_cores(local: Sequence[Sequence[torch.Tensor]], batch: int, device=None) -> List[List[torch.Tensor]]:
    """local: for each locally-owned problem, its list of TT cores.  Returns the cores of all `batch`
    problems on every rank.  Ranks are data dependent (eps-driven), so shapes (and the dtype) are gathered
    first, then one flat all-gather moves the payload (padded to the largest shard).  A rank that owns no
    problem (batch < world size) takes the dtype from the gathered metadata and the device from `device`
    (default: its current CUDA device under NCCL, the CPU under gloo)."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return [list(c) for c in local]
    world = dist.get_world_size()
    meta = dict(shapes=[[list(c.shape) for c in cores] for cores in local],
                dtype=_dtype_name(local[0][0].dtype) if len(local) else None)
    metas = [None] * world
    dist.all_gather_object(metas, meta)
    names = {m["dtype"] for m in metas if m["dtype"] is not None}
    if len(names) > 1:
        raise ValueError(f"all_gather_cores: ranks hold different dtypes {sorted(names)}")
    dtype = getattr(torch, names.pop()) if names else torch.float32
    if len(local):
        dev = local[0][0].device
    elif device is not None:
        dev = torch.device(device)
    elif dist.get_backend() == "nccl":
        dev = torch.device("cuda", torch.cuda.current_device())
    else:
        dev = torch.device("cpu")
    flat = torch.cat([c.reshape(-1) for cores in local for c in cores]) if len(local) else torch.empty(0, dtype=dtype, device=dev)
    sizes = [sum(int(torch.Size(s).numel()) for cores in m["shapes"] for s in cores) for m in metas]
    pad = max(max(sizes) if sizes else 0, 1)
    buf = torch.zeros(pad, dtype=dtype, device=dev)
    buf[: flat.numel()] = flat
    out = [torch.empty(pad, dtype=dtype, device=dev) for _ in range(world)]
    dist.all_gather(out, buf)
    result: List[List[torch.Tensor]] = []
    for g in range(world):
        off = 0
        for cores in metas[g]["shapes"]:
            cur = []
            for s in cores:
                n = int(torch.Size(s).numel())
                cur.append(out[g][off: off + n].view(*s))
                off += n
            result.append(cur)
    assert len(result) == batch, (len(result), batch)
    return result


def ttsvd_batch_sharded(tensors: Sequence[torch.Tensor], rmax=None, eps: float = 1e-14, gather: bool = True):
    """Decompose a batch of dense tensors, sharded over the ranks of the default process group."""
    from . import ops

    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    lo, hi = shard_range(len(tensors), world, rank)
    # the local shard goes through ONE library call (tnb_ttsvd_batch: several tensors in flight per GPU)
    local = ops.ttsvd_batch([tensors[i] for i in range(lo, hi)], rmax=rmax, eps=eps) if hi > lo else []
    return all_gather_cores(local, len(tensors)) if gather else local


def batch_sharded(problems: Sequence, solve, gather: bool = True):
    """The sharding pattern shared by every batched workload of the path (BASELINE.json configs 3-5): rank g solves
    the contiguous slice of `problems` it owns with `solve(problem) -> list of tensors` (TT cores or CP factors), no
    collective in between, then ONE all-gather of the ragged results."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    lo, hi = shard_range(len(problems), world, rank)
    local = [list(solve(problems[i])) for i in range(lo, hi)]
    return all_gather_cores(local, len(problems)) if gather else local


def round_tt_batch_sharded(tts: Sequence[Sequence[torch.Tensor]], rmax=None, eps: float = 1e-14, gather: bool = True):
    """config 3 in batch form: a list of TT tensors (lists of cores), each rounded on the rank that owns it."""
    from . import ops

    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    lo, hi = shard_range(len(tts), world, rank)
    same = hi > lo and all([c.shape for c in tts[i]] == [c.shape for c in tts[lo]] for i in range(lo, hi))
    if same:  # one library call for the local shard, several tensors in flight (tnb_tt_round_batch)
        local = ops.tt_round_batch([list(tts[i]) for i in range(lo, hi)], eps=eps, rmax=rmax)
    else:
        local = [ops.tt_round(list(tts[i]), eps=eps, rmax=rmax) for i in range(lo, hi)]
    return all_gather_cores(local, len(tts)) if gather else local


def cp_als_batch_sharded(tensors: Sequence[torch.Tensor], R: int, max_iter: int = 25, tol: float = 1e-4, gather: bool = True):
    """config 4 ("1 vs 8 GPUs batch-sharded"): independent CP-ALS problems, one per owned tensor."""
    from . import ops

    return batch_sharded(tensors, lambda X: ops.cp_als(X, R, max_iter=max_iter, tol=tol), gather)


def cross_batch_sharded(functions: Sequence, domain, gather: bool = True, **cross_kw):
    """config 5 (B black-box functions on the same grid, sharded over the GPUs).  With fixed ranks (`ranks_tt=`) the
    local shard advances as ONE batch (tntorch_b200.cross_batch: batched gather / QR / maxvol per sweep step); otherwise
    (adaptive ranks) it is `tn.cross` per owned function, like the reference, which has no batch support in `cross`
    (cross.py:256-258)."""
    from .cross import cross
    from .cross_batch import cross_batch

    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    lo, hi = shard_range(len(functions), world, rank)
    if cross_kw.get("ranks_tt") is not None and hi > lo:
        kw = {k: v for k, v in cross_kw.items() if k in ("ranks_tt", "eps", "max_iter", "val_size", "function_arg", "device")}
        t = cross_batch(list(functions[lo:hi]), domain, **kw)
        local = [[c[b] for c in t.cores] for b in range(hi - lo)]
    else:
        kw = dict(verbose=False, suppress_warnings=True)
        kw.update(cross_kw)
        local = [list(cross(functions[i], domain=domain, **kw).cores) for i in range(lo, hi)]
    return all_gather_cores(local, len(functions)) if gather else local
