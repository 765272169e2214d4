"""N ranks == 1 rank on the same global batch, through the Engine + Trainer + NCCL (needs >= 2 GPUs; skips on a
single-GPU machine)."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('mp', [False, True])
def test_two_rank_trainer_equals_single_process(mp, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    port = 29600 + os.getpid() % 1000
    env = dict(os.environ, DDP_TEST_MP='1' if mp else '0', NCCL_DEBUG='WARN', DDP_LOG_DIR=str(tmp_path))
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2', '--master-addr', '127.0.0.1',
                        '--master-port', str(port), os.path.join(ROOT, 'tests', 'ddp_worker.py')], capture_output=True, text=True,
                       env=env, timeout=240)
    line = next((l for l in r.stdout.splitlines() if l.startswith('DDP_RESULT ')), None)
    assert line is not None, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(line[len('DDP_RESULT '):])
    for case, v in res.items():
        # fp32: same kernels, same per-row arithmetic, only the summation order over rows differs (atomics / split-K);
        # bf16: dW accumulates bf16-rounded operands in a different grouping of rows
        assert abs(v['loss_ddp'] - v['loss_single']) < (2e-3 if mp else 1e-5), (case, v)
        assert v["grad_rel_l2"] < (1e-3 if mp else 1e-5), (case, v)
    assert res['even_4_rows_graph']['graph'], 'the data-parallel step was not captured into a CUDA graph'
    assert res['one_row_idle_rank']['shard_rows'] == 1
