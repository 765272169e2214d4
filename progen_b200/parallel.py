"""Data parallelism — the only parallelism the reference has (`pmap` over the batch, utils.py:69-91).

One process per GPU (torchrun), replicas keep parameters and optimizer state resident, the batch is split by rows and
the only exchange is a SUM all-reduce of the flat fp32 gradient buffer over NCCL (NVLink 5 / NVSwitch), plus one scalar
for the logged loss.  The reference pads a ragged batch to a multiple of the device count and takes a masked mean
(utils.py:83-91); here every rank scales its per-row losses by 1/global_rows so the SUM of the per-rank gradients is
exactly that masked mean — no padding rows are ever computed.
"""
import torch
import torch.distributed as dist


def world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_rows(num_rows, rank, world_size):
    """Row range of `rank` under the reference's '(p b) ... -> p b ...' split of a batch padded to a multiple of p
    (utils.py:83-89).  Returns (start, stop) into the UNPADDED batch; trailing ranks may get fewer (or zero) rows."""
    per = -(-num_rows // world_size)
    start = min(num_rows, rank * per)
    stop = min(num_rows, start + per)
    return start, stop


def shard_batch(data, rank=None, world_size=None):
    r, w = world()
    rank = r if rank is None else rank
    world_size = w if world_size is None else world_size
    a, b = shard_rows(data.shape[0], rank, world_size)
    return data[a:b]


def allreduce_scalar_(t, group=None):
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t
