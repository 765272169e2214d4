"""Worker of tests/test_gpu_ddp.py (one process per GPU, launched by torch.distributed.run): the data-parallel path of
Trainer.step through the real Engine and NCCL must reproduce the single-process gradient of the same GLOBAL batch —
reference utils.py:78-91 (pmap over a padded batch + masked mean).  Cases: ragged (5 rows over 2 ranks = 3 + 2), a rank
with no rows at all (1 row over 2 ranks), an even batch replayed through the captured CUDA graph."""
import json
import os
import tempfile
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    from progen_b200 import ProGen, parallel as PAR
    mp = os.environ.get('DDP_TEST_MP', '1') == '1'
    kwargs = dict(num_tokens=256, dim=128, seq_len=256, depth=2, window_size=128, global_mlp_depth=1, heads=2, dim_head=64)
    out = {}
    log_dir = os.environ.get('DDP_LOG_DIR') or tempfile.mkdtemp(prefix='progen_ddp_')
    os.makedirs(log_dir, exist_ok=True)
    log = open(os.path.join(log_dir, f'ddp_worker_mp{int(mp)}_rank{rank}.log'), 'w')

    def say(*a):
        print(f'[ddp_worker rank {rank}]', *a, file=log, flush=True)
    for case, rows in (('ragged_5_rows', 5), ('one_row_idle_rank', 1), ('even_4_rows_graph', 4)):
        say('case', case)
        data = np.random.default_rng(100 + rows).integers(0, 256, (rows, kwargs['seq_len'] + 1)).astype(np.int32)
        data[0, 100:] = 0
        model = ProGen(**kwargs, mixed_precision=mp)
        params = model.init(7)
        # lr = 0: the step leaves the parameters alone, so eng.grads after the step IS the exchanged gradient
        tr = model.trainer(params, learning_rate=0.0, weight_decay=0.0, data_parallel=True, cuda_graph=(case == 'even_4_rows_graph'))
        shard = PAR.shard_batch(data)
        steps = 4 if case == 'even_4_rows_graph' else 1           # two eager steps, capture, then replays
        for i_ in range(steps):
            loss = tr.step(shard, sync_loss=True, global_batch=rows)
            torch.cuda.synchronize()
            say('step', i_, 'done, graph =', tr._graph is not None)
        g_ddp = tr.eng.grads.clone()
        l_ddp = float(loss.item())
        used_graph = tr._graph is not None
        if rank == 0:
            single = ProGen(**kwargs, mixed_precision=mp)
            single.engine.load_params(params)
            l_one = float(single.engine.loss_and_grad(data).item())
            g_one = single.engine.grads
            den = float(g_one.norm().item())
            out[case] = dict(loss_ddp=l_ddp, loss_single=l_one, grad_rel_l2=float((g_ddp - g_one).norm().item()) / den,
                             grad_max_abs=float((g_ddp - g_one).abs().max().item()), grad_absmax=float(g_one.abs().max().item()),
                             graph=used_graph, world=world, shard_rows=int(shard.shape[0]))
        say('case done, entering barrier')
        dist.barrier()
        torch.cuda.synchronize()
        say('barrier passed')
    if rank == 0:
        print('DDP_RESULT ' + json.dumps(out), flush=True)
        say('DDP_RESULT ' + json.dumps(out))
    say('exiting')
    log.close()
    sys.stdout.flush()
    os._exit(0)      # no interpreter / NCCL teardown: captured graphs still reference the communicator


if __name__ == '__main__':
    main()
