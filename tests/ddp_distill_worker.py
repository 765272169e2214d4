"""Worker of tests/test_gpu_distill.py::test_two_rank_step (one process per GPU, launched by torch.distributed.run):
every rank holds its own teacher and a shard of the global batch (3 + 2 rows, so the shards are ragged) and runs the
distillation step at the global batch's cut length; the all-reduced gradient must equal the single-process step's on
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
    student_kw = dict(num_tokens=256, dim=128, seq_len=256, depth=2, window_size=64, global_mlp_depth=1, heads=2, dim_head=64)
    teacher_kw = dict(student_kw, dim=192, heads=3, depth=3, seq_len=320)
    n = student_kw['seq_len']
    data = np.random.default_rng(30).integers(1, 256, (5, n + 1)).astype(np.int32)
    for i, k in enumerate([200, 90, 20, 100, 60]):
        data[i, 1 + k:] = 0
    length = cut_length(data[:, 1:])
    out = {}
    for mp in (False, True):
        model, teacher = ProGen(**student_kw, mixed_precision=mp), ProGen(**teacher_kw, mixed_precision=mp)
        params, tparams = model.init(7), teacher.init(9)
        tr = model.trainer(params, learning_rate=0.0, weight_decay=0.0, data_parallel=True, teacher=teacher,
                           teacher_params=tparams)
        shard = PAR.shard_batch(data)
        loss = float(tr.distill_step(shard, 2.0, 0.5, sync_loss=True, global_batch=len(data), length=length).item())
        g_ddp = tr.eng.grads.clone()
        if rank == 0:
            single = ProGen(**student_kw, mixed_precision=mp)
            l_one, _, _ = single.distill_loss_and_grad(params, data, teacher=ProGen(**teacher_kw, mixed_precision=mp),
                                                       teacher_params=tparams)
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
