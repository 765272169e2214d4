"""Training with recomputed activations (DESIGN.md §3.12) against the resident training step.

    python scripts/recompute_bench.py [--steps 5] [--rounds 3]

Cases (bf16, ProGen.init(0), seeded uniform rows at full length, captured steps of Trainer(cuda_graph=True)):
  config 2, B = 64: the full fine-tune and LoRA r = 16, resident and recompute;
  config 4, B = 4: the full fine-tune, resident and recompute;
  config 4, B = 8 and 16: the full fine-tune in recompute mode (resident, the training set alone outgrows the card).
A mode runs only when its training set (`engine.training_set`, counted from the shapes) fits in the free memory
`torch.cuda.mem_get_info` reports with the model and optimizer state resident; nothing probes for an out-of-memory.
For each case and mode:
  step time: the median (min, max) over rounds of `steps` captured steps timed with CUDA events; in a case with both
    modes, one trainer alternates them round by round (`ProGen.recompute` re-allocates the training set, the step is
    captured again, outside the timed window);
  tokens/s: B * seq_len over the median step time;
  peak: torch's allocation peak over a fresh trainer's first steps, above what was allocated before its first step
    (parameters, gradients and optimizer state), against the training set's byte count.
Prints one JSON line with the card name and power limit."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, gpu_info                      # noqa: E402
from progen_b200 import ProGen                           # noqa: E402
from progen_b200.engine import training_set             # noqa: E402

GIB = 2 ** 30
CASES = [('cfg2', 64, 'full', (False, True)), ('cfg2', 64, 'lora_r16', (False, True)), ('cfg4', 4, 'full', (False, True)),
         ('cfg4', 8, 'full', (True,)), ('cfg4', 16, 'full', (True,))]


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def trainer(model, params, kind):
    kw = dict(adapters=model.init_adapters(0, 16)) if kind == 'lora_r16' else {}
    return model.trainer(params, cuda_graph=True, **kw)


def release():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def case(name, B, kind, modes, params, steps, rounds):
    kw = CONFIGS[name]['kwargs']
    n = kw['seq_len']
    cfg = ProGen(**kw).config
    rows = np.random.default_rng(42).integers(0, 256, (B, n + 1))
    out = dict(config=name, batch=B, kind=kind, modes={})
    fits = []
    for rc in modes:
        need = training_set(cfg, B, True, rc)[1]
        model = ProGen(**kw, mixed_precision=True, recompute=rc)
        tr = trainer(model, params, kind)
        release()
        free = torch.cuda.mem_get_info()[0]
        m = out['modes']['recompute' if rc else 'resident'] = dict(training_set_gib=round(need / GIB, 3),
                                                                   free_gib=round(free / GIB, 3))
        # the training set, plus a quarter for the step's transient buffers and the captured graph's pool
        if need * 1.25 > free:
            m['fits'] = False
        else:
            before = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            for _ in range(3):
                tr.step(rows)
            torch.cuda.synchronize()
            m.update(fits=True, peak_above_resident_gib=round((torch.cuda.max_memory_allocated() - before) / GIB, 3))
            fits.append(rc)
        del tr, model
        release()
    if not fits:
        return out
    model = ProGen(**kw, mixed_precision=True, recompute=fits[0])
    tr = trainer(model, params, kind)
    times = {rc: [] for rc in fits}
    for _ in range(rounds):
        for rc in fits:                                  # both modes alternate in one trainer
            model.recompute = rc
            for _ in range(3):                           # two eager steps and the capture of this allocation
                tr.step(rows)
            times[rc].append(timed(lambda: tr.step(rows), steps))
    for rc in fits:
        t = times[rc]
        med = statistics.median(t)
        out['modes']['recompute' if rc else 'resident'].update(
            step_ms=dict(median=round(med, 3), min=round(min(t), 3), max=round(max(t), 3)),
            tokens_per_s=round(B * n / (med / 1e3)))
    if len(fits) == 2:
        out['recompute_over_resident'] = round(statistics.median(times[True]) / statistics.median(times[False]), 4)
    del tr, model
    release()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    res = dict(gpu=gpu_info(torch.cuda.current_device()), steps=args.steps, rounds=args.rounds, cases=[])
    params = {}
    for name, B, kind, modes in CASES:
        if name not in params:
            params = {name: ProGen(**CONFIGS[name]['kwargs']).init(0)}          # one config's parameters at a time
        res['cases'].append(case(name, B, kind, modes, params[name], args.steps, args.rounds))
        print(json.dumps(res['cases'][-1]), file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
