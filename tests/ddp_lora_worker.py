"""Worker of tests/test_gpu_lora.py::test_two_rank_lora_trainer_equals_single_process (one process per GPU, launched by
torch.distributed.run): data-parallel adapter training must reproduce one process on the same GLOBAL batch.  Cases: a
ragged batch (5 rows over 2 ranks = 3 + 2) in eager steps, and an even batch through the captured CUDA graph (two eager
steps, the capture, then replays).  Compared on rank 0: the losses, the last step's (all-reduced) adapter gradient and
the adapters after the steps."""
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
    for case, rows, steps, graph in (('ragged_5_rows', 5, 2, False), ('even_4_rows_graph', 4, 4, True)):
        batches = []
        for s in range(steps):
            d = np.random.default_rng(100 * rows + s).integers(0, 256, (rows, kwargs['seq_len'] + 1)).astype(np.int32)
            d[0, 100:] = 0
            batches.append(d)
        model = ProGen(**kwargs, mixed_precision=mp)
        params = model.init(7)
        ad = model.init_adapters(3, 16, alpha=32.0)
        rng = np.random.default_rng(5)
        for v in ad.values():
            v['lora_b'] = (0.05 * rng.standard_normal(v['lora_b'].shape)).astype(np.float32)
        opt = dict(adapters=ad, lora_alpha=32.0, learning_rate=1e-2, grad_accum_every=1)
        tr = model.trainer(params, data_parallel=True, cuda_graph=graph, **opt)
        losses = [float(tr.step(PAR.shard_batch(d), sync_loss=True, global_batch=rows).item()) for d in batches]
        torch.cuda.synchronize()
        g_ddp, a_ddp, used_graph = tr.lora.grads.clone(), tr.adapters(), tr._graph is not None
        if rank == 0:
            one = ProGen(**kwargs, mixed_precision=mp).trainer(params, data_parallel=False, **opt)
            l_one = [float(one.step(d).item()) for d in batches]
            g_one, a_one = one.lora.grads, one.adapters()
            num = sum(float(np.linalg.norm(a_ddp[m][k] - a_one[m][k])) ** 2 for m in a_one for k in a_one[m]) ** 0.5
            den = sum(float(np.linalg.norm(a_one[m][k])) ** 2 for m in a_one for k in a_one[m]) ** 0.5
            out[case] = dict(loss_ddp=losses, loss_single=l_one, graph=used_graph,
                             grad_rel_l2=float((g_ddp - g_one).norm().item()) / float(g_one.norm().item()),
                             adapter_rel_l2=num / den)
        dist.barrier()
        torch.cuda.synchronize()
    if rank == 0:
        print('DDP_RESULT ' + json.dumps(out), flush=True)
    sys.stdout.flush()
    os._exit(0)      # no interpreter / NCCL teardown: captured graphs still reference the communicator


if __name__ == '__main__':
    main()
