"""Data-parallel plumbing (SURVEY.md §8e): shard DIALOGS across ranks (never split a dialog: the 10
rounds of a dialog are coupled by the history attention), one NCCL communicator inside the engine for
the single gradient all-reduce, rank-ordered gather of eval results.  torch.distributed is used only
for the out-of-band exchange (unique id, timing max, result gather); the reference is single-GPU
(train.lua:15-21)."""
from __future__ import annotations

from typing import Callable, Dict, Optional

import numpy as np


def shard_range(B: int, rank: int, world: int):
    base, rem = divmod(B, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(batch: Dict[str, np.ndarray], rank: int, world: int, rounds: int = 10) -> Dict[str, np.ndarray]:
    B = batch["ques_fwd"].shape[0]
    lo, hi = shard_range(B, rank, world)
    out = {}
    for k, v in batch.items():
        if v.shape[0] == B:
            out[k] = v[lo:hi]
        elif v.shape[0] == B * rounds:                       # options / answer_ind are (B*10, ...)
            out[k] = v[lo * rounds:hi * rounds]
        else:
            raise ValueError("cannot shard %s with leading dim %d" % (k, v.shape[0]))
    return out


def broadcast_unique_id(make_id: Callable[[], Optional[bytes]], rank: int) -> bytes:
    import torch
    import torch.distributed as dist
    buf = torch.zeros(128, dtype=torch.uint8)
    if rank == 0:
        buf = torch.frombuffer(bytearray(make_id()), dtype=torch.uint8).clone()
    if dist.get_backend() == "nccl":
        buf = buf.cuda()
    dist.broadcast(buf, src=0)
    return bytes(buf.cpu().numpy().tobytes())


def gather_ranks(local: np.ndarray, rank: int, world: int) -> Optional[np.ndarray]:
    import torch.distributed as dist
    objs = [None] * world
    dist.all_gather_object(objs, local)
    return np.concatenate(objs, 0)


def gather_objects(local: list, world: int) -> list:
    """Rank-ordered concatenation of every rank's list (evaluation tables, generated dialogs)."""
    import torch.distributed as dist
    objs = [None] * world
    dist.all_gather_object(objs, local)
    return [x for part in objs for x in part]


def broadcast_object(obj, rank: int):
    """Rank 0's `obj` on every rank (a decision rank 0 took, such as ending training early)."""
    import torch.distributed as dist
    box = [obj if rank == 0 else None]
    dist.broadcast_object_list(box, src=0)
    return box[0]


def mean_over_ranks(value: float, world: int) -> float:
    import torch
    import torch.distributed as dist
    t = torch.tensor([value], dtype=torch.float64)
    if dist.get_backend() == "nccl":
        t = t.cuda()
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item()) / world


def max_over_ranks(value: float) -> float:
    import torch
    import torch.distributed as dist
    t = torch.tensor([value], dtype=torch.float64)
    if dist.get_backend() == "nccl":
        t = t.cuda()
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def attach_engine(engine, rank: int, world: int):
    """Create the engine's NCCL communicator: rank 0 makes the id, torch.distributed carries it."""
    if world <= 1:
        return
    uid = broadcast_unique_id(engine.comm_unique_id, rank)
    engine.comm_init(uid, rank, world)
