"""Host-side data-parallel logic on CPU with the gloo backend, world_size 2 (the N>1 path of bench.py / train.py):
row sharding follows the reference's '(p b)' split with ragged batches (utils.py:78-91), and a SUM all-reduce of
per-rank gradients scaled by 1/global_rows equals the single-process gradient of the masked mean."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shard_rows_covers_batch_like_reference_padding():
    from progen_b200.parallel import shard_rows
    for rows in range(1, 20):
        for world in (1, 2, 3, 4, 8):
            spans = [shard_rows(rows, r, world) for r in range(world)]
            got = [i for a, b in spans for i in range(a, b)]
            assert got == list(range(rows))
            per = -(-rows // world)
            assert all(b - a <= per for a, b in spans)


def _worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from progen_b200 import parallel as PAR
    from oracle import progen_ref as O
    from oracle import progen_torch as T
    torch.set_num_threads(2)
    kwargs = dict(num_tokens=256, dim=32, seq_len=16, depth=2, window_size=8, global_mlp_depth=1, heads=2, dim_head=16)
    cfg = O.make_config(**kwargs)
    params = O.randomize_params(O.init_params(cfg, 1), 2)
    data = np.random.default_rng(3).integers(0, 256, (5, cfg['seq_len'] + 1)).astype(np.int64)     # ragged: 5 rows / 2 ranks
    local = PAR.shard_batch(data)
    assert PAR.world() == (rank, world)
    # per-rank: sum of per-row losses / global_rows  (what Engine.loss_and_grad(global_batch=...) computes)
    prm = T.to_torch(params, torch.float64, requires_grad=True)
    ids, labels = torch.as_tensor(local[:, :-1]), torch.as_tensor(local[:, 1:])
    loss = T.cross_entropy(T.forward(prm, ids, cfg), labels).sum() / data.shape[0]
    loss.backward()
    keys = sorted((m, k) for m, d in prm.items() for k in d)
    flat = torch.cat([prm[m][k].grad.reshape(-1) for m, k in keys])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM)          # the exchange Trainer makes
    lt = PAR.allreduce_scalar_(loss.detach().clone())
    if rank == 0:
        ref_loss, ref = T.loss_and_grads(params, data, cfg)
        ref_flat = np.concatenate([ref[m][k].ravel() for m, k in keys])
        ret['loss_err'] = abs(float(lt) - ref_loss)
        ret['grad_err'] = float(np.abs(flat.numpy() - ref_flat).max())
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gloo_allreduce_equals_single_process_gradient():
    port = 29500 + (os.getpid() % 2000)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, port, ret), nprocs=2, join=True)
    assert ret['loss_err'] < 1e-12 and ret['grad_err'] < 1e-12, dict(ret)

