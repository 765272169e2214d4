"""Worker of tests/test_gpu_preference.py's data-parallel test (one process per GPU, launched by torch.distributed.run):
Trainer.preference_step over pairs sharded with parallel.shard_rows must reproduce the single-process loss and gradient of
all the pairs.  Cases: 5 pairs over 2 ranks (3 + 2) and 1 pair over 2 ranks (a rank without pairs)."""
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
    mp = os.environ.get('DDP_TEST_MP', '1') == '1'
    kwargs = dict(num_tokens=256, dim=128, seq_len=256, depth=2, window_size=128, global_mlp_depth=1, heads=2, dim_head=64)
    out = {}
    for case, P in (('ragged_5_pairs', 5), ('one_pair_idle_rank', 1)):
        rng = np.random.default_rng(200 + P)
        c = rng.integers(1, 256, (P, kwargs['seq_len'] + 1)).astype(np.int32)
        r = rng.integers(1, 256, (P, kwargs['seq_len'] + 1)).astype(np.int32)
        c[0, 100:] = 0
        model = ProGen(**kwargs, mixed_precision=mp)
        params = model.init(7)
        sc = model.score(params, np.concatenate([c, r]))['log_likelihood']
        ref_c, ref_r = sc[:P] + rng.normal(0, 3, P).astype(np.float32), sc[P:] + rng.normal(0, 3, P).astype(np.float32)
        # lr = 0: the step leaves the parameters alone, so eng.grads after the step IS the exchanged gradient
        tr = model.trainer(params, learning_rate=0.0, weight_decay=0.0, data_parallel=True)
        a, b = PAR.shard_rows(P, rank, dist.get_world_size())
        loss = tr.preference_step(c[a:b], r[a:b], ref_c[a:b], ref_r[a:b], beta=0.1, sync_loss=True, global_pairs=P)
        torch.cuda.synchronize()
        g_ddp, l_ddp = tr.eng.grads.clone(), float(loss.item())
        if rank == 0:
            single = ProGen(**kwargs, mixed_precision=mp)
            l_one, _, _ = single.preference_loss_and_grad(params, c, r, ref_c, ref_r, beta=0.1)
            g_one = single.engine.grads
            out[case] = dict(loss_ddp=l_ddp, loss_single=l_one,
                             grad_rel_l2=float((g_ddp - g_one).norm().item()) / float(g_one.norm().item()),
                             shard_pairs=b - a)
        dist.barrier()
        torch.cuda.synchronize()
    if rank == 0:
        print('DDP_RESULT ' + json.dumps(out), flush=True)
    sys.stdout.flush()
    os._exit(0)      # no interpreter / NCCL teardown


if __name__ == '__main__':
    main()
