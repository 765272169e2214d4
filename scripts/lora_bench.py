"""Cost of low-rank adapter (LoRA) fine-tuning against the full fine-tune it replaces, at the config-2 and config-4 shapes.

    python scripts/lora_bench.py [--rank 16] [--steps 10] [--rounds 3] [--cfg4_batches 8,4] [--skip_cfg4]

For each shape, one Trainer per mode (full: every parameter; lora: rank-r adapters on the four projections of every
layer, frozen base) on ProGen.init(0) and uniform-random rows from seed 42 (data.synthetic_iterator).  The step is
captured into a CUDA graph after two eager steps; a round times `steps` replays between CUDA events, and the median over
`rounds` rounds is reported.  When both trainers fit on the device together (config 2) their rounds alternate in one
process; otherwise (config 4) each mode is timed while it is the only one resident.  Peak device memory is torch's
allocation peak of one mode, from model construction through the capture and one replay, above what was resident
before it.  Checkpoint bytes are the array payload of what train.py stores: params, mu, nu, acc (full) or
adapters, mu, nu, acc (lora).  Config 2 runs at the benchmark's batch of 64 rows; config 4 at the first batch of
--cfg4_batches at which both modes fit.  Prints one JSON line with the card name and power limit."""
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


def tree_bytes(*trees):
    return int(sum(np.asarray(a).nbytes for t in trees for d in t.values() for a in d.values()))


def make(kw, params, batch, rank, lora):
    """a trainer of one mode with its step captured -> (trainer, model, peak device memory of the mode in GiB: the
    allocation peak from construction through two eager steps, the capture and one replay, above what was resident)"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    model = ProGen(**kw, mixed_precision=True)
    tr = model.trainer(params, adapters=model.init_adapters(0, rank) if lora else None)
    data = next(synthetic_iterator(kw['seq_len'], batch, seed=42))
    for _ in range(2):
        tr.step(data)
    tr.capture_graph(batch)
    tr.eng.load_batch(data)
    tr.step_resident()
    torch.cuda.synchronize()
    return tr, model, (torch.cuda.max_memory_allocated() - before) / 2 ** 30


def timed_round(tr, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        tr.step_resident()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def summary(tr, model, lora, peak, times):
    st = tr.optim_state()
    return dict(step_ms=statistics.median(times), step_ms_rounds=times, peak_mem_gib=peak,
                checkpoint_bytes=tree_bytes(tr.adapters() if lora else tr.params(), st['mu'], st['nu'], st['acc']),
                trained_params=tr.lora.num_params if lora else model.engine.num_params, loss=float(tr.eng.loss.item()))


def free():
    gc.collect()
    torch.cuda.empty_cache()


def shape(name, kw, params, batches, rank, steps, rounds):
    """both modes at the first batch that fits them; the rounds alternate full and LoRA when both trainers fit on the
    device together, else each mode's rounds run while it is the only one resident"""
    for batch in batches:
        full = lo = None
        try:
            full = make(kw, params, batch, rank, False)
            try:
                lo = make(kw, params, batch, rank, True)
            except torch.cuda.OutOfMemoryError:
                lo = None
            alternated = lo is not None
            if alternated:
                tf, tl = [], []
                for _ in range(rounds):
                    tf.append(timed_round(full[0], steps))
                    tl.append(timed_round(lo[0], steps))
                res_full, res_lora = summary(*full[:2], False, full[2], tf), summary(*lo[:2], True, lo[2], tl)
            else:
                free()                                 # what the failed second trainer had allocated
                res_full = summary(*full[:2], False, full[2], [timed_round(full[0], steps) for _ in range(rounds)])
                full = None
                free()
                lo = make(kw, params, batch, rank, True)
                res_lora = summary(*lo[:2], True, lo[2], [timed_round(lo[0], steps) for _ in range(rounds)])
        except (torch.cuda.OutOfMemoryError, L.ProgenError) as e:
            print(f'{name} batch {batch}: {type(e).__name__}: {str(e)[:200]}', file=sys.stderr)
            full = lo = None
            free()
            continue
        full = lo = None
        free()
        return dict(config=name, batch=batch, rank=rank, alternated=alternated, full=res_full, lora=res_lora,
                    speedup=res_full['step_ms'] / res_lora['step_ms'],
                    memory_ratio=res_lora['peak_mem_gib'] / res_full['peak_mem_gib'])
    return dict(config=name, error=f'no batch of {batches} fits both modes')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rank', type=int, default=16)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--cfg4_batches', default='8,4')
    ap.add_argument('--skip_cfg4', action='store_true')
    args = ap.parse_args()
    L.require_device()
    res = dict(gpu=gpu_info(torch.cuda.current_device()), results=[])
    kw2 = CONFIGS['cfg2']['kwargs']
    res['results'].append(shape('cfg2', kw2, ProGen(**kw2).init(0), [CONFIGS['cfg2']['batch']], args.rank, args.steps,
                                args.rounds))
    if not args.skip_cfg4:
        kw4 = CONFIGS['cfg4']['kwargs']
        batches = [int(b) for b in args.cfg4_batches.split(',')]
        res['results'].append(shape('cfg4', kw4, ProGen(**kw4).init(0), batches, args.rank, args.steps, args.rounds))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
