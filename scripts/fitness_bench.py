"""Cost of a property fine-tuning step (head on the pooled embedding, rank-r adapters, frozen base) against the LoRA
language-model step on the same rows, at the config-2 and config-4 shapes.

    python scripts/fitness_bench.py [--rank 16] [--steps 10] [--rounds 3] [--cfg4_batch 4] [--skip_cfg4]

For each shape, one trainer per mode on ProGen.init(0), the same adapters (rank r, seed 0) and the same uniform-random
rows (seed 42, data.synthetic_iterator); the property head is a 3-output regression head with standard-normal targets.
Each step is captured into a CUDA graph after two eager steps; a round times `steps` replays between CUDA events and the
median over `rounds` rounds is reported.  When both trainers fit on the device together their rounds alternate;
otherwise each mode is timed while it is the only one resident.  Peak device memory is torch's allocation peak of one
mode, from model construction through the capture and one replay, above what was resident before it.  The share of the
property step spent in progen_property_head's two kernels and in progen_masked_mean_pool_bwd comes from a separate
torch.profiler run of `steps` replays (kernel time over the summed kernel time of the step).  Prints one JSON line with
the card name and power limit."""
import argparse
import gc
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, gpu_info                      # noqa: E402
from progen_b200 import ProGen, lib as L                 # noqa: E402
from progen_b200.data import synthetic_iterator          # noqa: E402

HEAD_KERNELS = ('property_head_rows_kernel', 'property_head_params_kernel', 'masked_mean_pool_bwd_kernel')


def make(kw, params, rows, targets, rank, prop):
    """a trainer of one mode with its step captured -> (replay function, trainer, peak memory of the mode in GiB)"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    model = ProGen(**kw, mixed_precision=True)
    ad = model.init_adapters(0, rank)
    if prop:
        tr = model.trainer(params, adapters=ad, head=model.init_head(0, targets.shape[1]), task='regression', cuda_graph=True)
        for _ in range(3):                                # two eager steps, the capture, then one replay
            tr.property_step(rows, targets)
        replay = tr._replay
    else:
        tr = model.trainer(params, adapters=ad, cuda_graph=True)
        for _ in range(3):
            tr.step(rows)
        replay = tr.step_resident
    assert tr._graph is not None
    torch.cuda.synchronize()
    return replay, tr, (torch.cuda.max_memory_allocated() - before) / 2 ** 30


def timed_round(replay, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def head_share(replay, steps):
    """fraction of the step's kernel time in the property head and pool-backward kernels, and their time per step (us)"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            replay()
        torch.cuda.synchronize()
    total = head = 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
        if e.key.startswith('ProfilerStep') or t <= 0:
            continue
        total += t
        if any(k in e.key for k in HEAD_KERNELS):
            head += t
    return head / max(total, 1e-9), head / steps


def free():
    gc.collect()
    torch.cuda.empty_cache()


def shape(name, kw, batch, rank, steps, rounds):
    params = ProGen(**kw).init(0)
    rows = next(synthetic_iterator(kw['seq_len'], batch, seed=42))
    targets = np.random.default_rng(0).standard_normal((batch, 3)).astype(np.float32)
    lm = pr = None
    try:
        lm = make(kw, params, rows, targets, rank, False)
        try:
            pr = make(kw, params, rows, targets, rank, True)
        except torch.cuda.OutOfMemoryError:
            pr = None
        alternated = pr is not None
        if alternated:
            tl, tp = [], []
            for _ in range(rounds):
                tl.append(timed_round(lm[0], steps))
                tp.append(timed_round(pr[0], steps))
        else:
            free()
            tl = [timed_round(lm[0], steps) for _ in range(rounds)]
            lm_peak = lm[2]
            lm = None
            free()
            pr = make(kw, params, rows, targets, rank, True)
            tp = [timed_round(pr[0], steps) for _ in range(rounds)]
        share, head_us = head_share(pr[0], steps)
        res = dict(config=name, batch=batch, rank=rank, alternated=alternated,
                   lm_step_ms=statistics.median(tl), lm_step_ms_rounds=tl,
                   property_step_ms=statistics.median(tp), property_step_ms_rounds=tp,
                   lm_peak_mem_gib=lm[2] if lm is not None else lm_peak, property_peak_mem_gib=pr[2],
                   head_and_pool_bwd_share=share, head_and_pool_bwd_us_per_step=head_us,
                   property_loss=float(pr[1].eng.loss.item()))
        res['property_over_lm'] = res['property_step_ms'] / res['lm_step_ms']
        return res
    except (torch.cuda.OutOfMemoryError, L.ProgenError) as e:
        return dict(config=name, batch=batch, error=f'{type(e).__name__}: {str(e)[:200]}')
    finally:
        lm = pr = None
        free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rank', type=int, default=16)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--cfg4_batch', type=int, default=4)
    ap.add_argument('--skip_cfg4', action='store_true')
    args = ap.parse_args()
    L.require_device()
    res = dict(gpu=gpu_info(torch.cuda.current_device()), results=[])
    res['results'].append(shape('cfg2', CONFIGS['cfg2']['kwargs'], CONFIGS['cfg2']['batch'], args.rank, args.steps,
                                args.rounds))
    if not args.skip_cfg4:
        res['results'].append(shape('cfg4', CONFIGS['cfg4']['kwargs'], args.cfg4_batch, args.rank, args.steps, args.rounds))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
