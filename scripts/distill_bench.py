"""Distillation (DESIGN.md §3.13) against the student's LM step.

    python scripts/distill_bench.py [--steps 5] [--rounds 3]

Cases (bf16, ProGen.init(0) for student and teacher, seeded uniform rows at the student's full length, 1024): a config-4
teacher into a config-2 student at B = 16 and 64, and a config-3 teacher into a config-2 student at B = 64.  The teacher
runs at L_t = 1024 (a multiple of 128 below its seq_len).  For each case:
  step_ms: the median (min, max) over rounds of `steps` captured steps (Trainer(cuda_graph=True)) timed with CUDA events,
    the distillation step and the student's LM step alternating round by round in one trainer;
  teacher_ms: the teacher's forward alone on its (B, L_t) view (eager launches, CUDA events), and its share of the step;
  head_ms: progen_distill_head alone, against its HBM floor T V (4 + 4 + 2) bytes / 3.35 TB/s (student logits, teacher
    logits and bf16 dlogits; the data-sheet bandwidth of the H100 SXM);
  peak_gib: torch's allocation peak over the first distillation steps, above what the trainer and teacher held before.
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
from progen_b200 import lib as L                         # noqa: E402
from progen_b200.distill import teacher_length           # noqa: E402

GIB = 2 ** 30
HBM_BYTES_PER_S = 3.35e12
CASES = [('cfg4', 'cfg2', 16), ('cfg4', 'cfg2', 64), ('cfg3', 'cfg2', 64)]
TAU, ALPHA = 2.0, 0.5


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def stat(t):
    return dict(median=round(statistics.median(t), 3), min=round(min(t), 3), max=round(max(t), 3))


def case(tname, sname, B, steps, rounds):
    skw, tkw = CONFIGS[sname]['kwargs'], CONFIGS[tname]['kwargs']
    n = skw['seq_len']
    student, teacher = ProGen(**skw, mixed_precision=True), ProGen(**tkw, mixed_precision=True)
    rows = np.random.default_rng(42).integers(1, 256, (B, n + 1))
    tr = student.trainer(student.init(0), cuda_graph=True, teacher=teacher, teacher_params=teacher.init(0))
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(3):                                   # two eager steps and the capture
        tr.distill_step(rows, TAU, ALPHA)
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - before) / GIB
    for _ in range(3):
        tr.step(rows)
    times = dict(distill=[], lm=[])
    for _ in range(rounds):
        times['distill'].append(timed(lambda: tr.distill_step(rows, TAU, ALPHA), steps))
        times['lm'].append(timed(lambda: tr.step(rows), steps))
    eng, te = tr.eng, teacher.engine
    Lt = teacher_length(n, te.n)
    ta = te.infer.view(B, Lt)
    teacher_ms = [timed(lambda: te._forward_device(ta), steps) for _ in range(rounds)]
    eng.load_distill(rows, n)
    a = eng.acts
    g = a.grad
    lib, st = L.load(), L.stream()

    def head():
        L.check(lib.progen_distill_head(a.logits.data_ptr(), L.F32, ta.logits.data_ptr(), Lt, a.labels.data_ptr(),
                                        g['ce_w'].data_ptr(), eng.dist['scratch'].data_ptr(), eng.dist['stats'].data_ptr(),
                                        eng.loss.data_ptr(), g['dlogits'].data_ptr(), eng.act_dt, B, n, eng.V, TAU, ALPHA,
                                        1.0 / B, st), 'distill_head')
    head()
    head_ms = [timed(head, 20 * steps) for _ in range(rounds)]
    floor_ms = B * n * eng.V * (4 + 4 + 2) / HBM_BYTES_PER_S * 1e3
    d, lm, t, h = (statistics.median(x) for x in (times['distill'], times['lm'], teacher_ms, head_ms))
    out = dict(teacher=tname, student=sname, batch=B, teacher_length=Lt, step_ms=dict(distill=stat(times['distill']),
               lm=stat(times['lm'])), distill_over_lm=round(d / lm, 4), teacher_ms=stat(teacher_ms),
               teacher_share=round(t / d, 4), head_ms=stat(head_ms), head_floor_ms=round(floor_ms, 4),
               head_over_floor=round(h / floor_ms, 2), head_share=round(h / d, 4), peak_gib=round(peak, 3))
    del tr, student, teacher
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    res = dict(gpu=gpu_info(torch.cuda.current_device()), steps=args.steps, rounds=args.rounds, cases=[])
    for tname, sname, B in CASES:
        res['cases'].append(case(tname, sname, B, args.steps, args.rounds))
        print(json.dumps(res['cases'][-1]), file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
