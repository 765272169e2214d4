"""Worker of tests/test_gpu_policy.py::test_two_rank_step (one process per GPU, launched by torch.distributed.run): every
rank holds its own reference and a shard of the global batch (3 + 2 rows, so the shards are ragged) and runs the
policy-gradient step at the global batch's cut length; the all-reduced gradient must equal the single-process step's on
the global batch.  Writes {mp: result} as JSON to argv[1] (rank 0)."""
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
    kw = dict(num_tokens=256, dim=128, seq_len=256, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)
    n = kw['seq_len']
    data = np.random.default_rng(30).integers(1, 256, (5, n + 1)).astype(np.int32)
    lengths = [200, 90, 20, 100, 60]
    for i, k in enumerate(lengths):
        data[i, 1 + k:] = 0
    span = np.array([[3, 201], [0, 91], [5, 21], [50, 101], [1, 2]], np.int32)
    adv = np.array([0.5, -1.0, 0.25, 1.5, -0.75], np.float32)
    length = cut_length(data[:, 1:])
    out = {}
    for mp in (False, True):
        model, ref = ProGen(**kw, mixed_precision=mp), ProGen(**kw, mixed_precision=mp)
        params, rparams = model.init(7), model.init(9)
        tr = model.trainer(params, learning_rate=0.0, weight_decay=0.0, data_parallel=True, reference=ref,
                           reference_params=rparams)
        idx = PAR.shard_batch(np.arange(len(data)))
        loss = float(tr.policy_step(data[idx], span[idx], adv[idx], 0.1, sync_loss=True, global_rows=len(data),
                                    length=length).item())
        g_ddp = tr.eng.grads.clone()
        if rank == 0:
            single = ProGen(**kw, mixed_precision=mp)
            l_one, _, _ = single.policy_loss_and_grad(params, data, adv, reference=ProGen(**kw, mixed_precision=mp),
                                                      reference_params=rparams, beta=0.1, span=span)
            g_one = single.engine.grads
            out[str(mp)] = dict(loss_ddp=loss, loss_single=l_one, length=int(length),
                                grad_rel_l2=float((g_ddp - g_one).norm().item()) / float(g_one.norm().item()))
        dist.barrier()
        torch.cuda.synchronize()
    if rank == 0:
        with open(sys.argv[1], 'w') as f:
            json.dump(out, f)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
