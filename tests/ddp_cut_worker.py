"""Worker of tests/test_gpu_cut_train.py::test_two_rank_cut_step_equals_single_process (one process per GPU, launched by
torch.distributed.run): every rank holds the global micro-batch, takes its shard and runs the step at the cut length of
the global batch (`engine.cut_length`), as train.py does.  The shards' own cut lengths differ; every rank runs the one
global length, so the collectives pair up.  The all-reduced gradient must equal the single-process step's on the global
batch.  Writes {mp: result} as JSON to argv[1] (rank 0)."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, local = int(os.environ['RANK']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    from progen_b200 import ProGen, parallel as PAR
    from progen_b200.engine import cut_length
    kwargs = dict(num_tokens=256, dim=128, seq_len=512, depth=2, window_size=256, global_mlp_depth=1, heads=2, dim_head=64)
    n = kwargs['seq_len']
    data = np.random.default_rng(30).integers(1, 256, (4, n + 1)).astype(np.int32)
    for i, k in enumerate([300, 350, 20, 100]):         # shards (2 + 2 rows): cut lengths 384 and 128
        data[i, 1 + k:] = 0
    length = cut_length(data[:, 1:])
    out = {}
    for mp in (False, True):
        model = ProGen(**kwargs, mixed_precision=mp)
        params = model.init(7)
        # lr = 0: the step leaves the parameters alone, so the gradient after the step IS the exchanged one
        tr = model.trainer(params, learning_rate=0.0, weight_decay=0.0, data_parallel=True)
        shard = PAR.shard_batch(data)
        loss = float(tr.step(shard, sync_loss=True, global_batch=len(data), length=length).item())
        g_ddp = tr.eng.grads.clone()
        lens = [None, None]
        dist.all_gather_object(lens, cut_length(shard[:, 1:]))
        if rank == 0:
            single = ProGen(**kwargs, mixed_precision=mp)
            single.engine.load_params(params)
            l_one = float(single.engine.loss_and_grad(data).item())
            g_one = single.engine.grads
            out[str(mp)] = dict(loss_ddp=loss, loss_single=l_one, length=int(length), shard_lengths=lens,
                                grad_rel_l2=float((g_ddp - g_one).norm().item()) / float(g_one.norm().item()))
        dist.barrier()
        torch.cuda.synchronize()
    if rank == 0:
        with open(sys.argv[1], 'w') as f:
            json.dump(out, f)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
