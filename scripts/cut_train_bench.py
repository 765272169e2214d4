"""The training step cut to its rows' counted length (DESIGN.md §3.10) against the full-length step, at config 2.

    python scripts/cut_train_bench.py [--steps 5] [--rounds 3] [--loop_batches 12]

Config 2 (d 512, depth 12, n 1024, window 256, bf16), B = 64, ProGen.init(0), one Trainer with cuda_graph=True.
1. Per-length step time: rows of counted length exactly L (seeded residues, then pad) for L = 128, 256, ..., 1024.  Each
   round times `steps` captured steps of `step(rows)` (at L) and then `steps` of `step(rows, length=n)` on the same rows
   (CUDA events, H2D copy of the rows included); rounds alternate over the lengths, and medians with min / max over the
   rounds are reported.  Also the LoRA (r = 16) step and the property step (3-output regression head, r = 16) at L = 384.
2. Peak memory: torch's allocation peak over the cut steps and over the full steps (after the captures).
3. Training loop: a train.py-shaped loop (batch 16, grad_accum_every 4, --loop_batches effective batches) on a seeded
   synthetic corpus whose lengths are log-normal with median 300 residues, clipped to [30, 1000] (not UniRef: nothing is
   downloaded), with and without data.group_by_length, eager and captured: counted tokens/s on the host clock (a
   device synchronise ends every timed loop).
Prints one JSON line with the card name and power limit."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, gpu_info                      # noqa: E402
from progen_b200 import ProGen                           # noqa: E402
from progen_b200.data import collate, group_by_length    # noqa: E402
from progen_b200.engine import counted_length            # noqa: E402


def rows_of_length(B, n, L, seed):
    """(B, n+1) rows of counted length exactly L: L - 1 residues after the BOS, then pad"""
    r = np.zeros((B, n + 1), np.uint16)
    r[:, 1:L] = np.random.default_rng(seed).integers(1, 256, (B, L - 1))
    return r


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def summary(xs):
    return dict(median_ms=round(statistics.median(xs), 3), min_ms=round(min(xs), 3), max_ms=round(max(xs), 3))


def per_length(tr, step, n, lengths, B, steps, rounds):
    """{L: {cut, full, speedup}} of step(rows, length) -> loss, alternated within each round"""
    rows = {L: rows_of_length(B, n, L, L) for L in lengths}
    for L in lengths:                                    # two eager steps and the capture of each (key, length)
        for _ in range(3):
            step(rows[L], None)
            step(rows[L], n)
    torch.cuda.synchronize()
    t = {L: dict(cut=[], full=[]) for L in lengths}
    for _ in range(rounds):
        for L in lengths:
            t[L]['cut'].append(timed(lambda: step(rows[L], None), steps))
            t[L]['full'].append(timed(lambda: step(rows[L], n), steps))
    out = {}
    for L in lengths:
        c, f = summary(t[L]['cut']), summary(t[L]['full'])
        out[L] = dict(cut=c, full=f, speedup=round(f['median_ms'] / c['median_ms'], 3))
    return out, rows


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round(torch.cuda.max_memory_allocated() / 2 ** 30, 3)


def corpus(count, seed=0):
    g = np.random.default_rng(seed)
    lens = np.clip(np.round(g.lognormal(np.log(300), 0.6, count)), 30, 1000).astype(int)
    aa = np.array(list('ACDEFGHIKLMNPQRSTVWY'))
    return [''.join(aa[g.integers(0, 20, k)]) for k in lens]


def loop(kw, params, seqs, grouped, graph, batch=16, every=4):
    """counted tokens/s of a train.py-shaped loop over seqs (a warm-up pass over the first two effective batches first)"""
    model = ProGen(**kw, mixed_precision=True)
    tr = model.trainer(params, grad_accum_every=every, cuda_graph=graph)
    n = kw['seq_len']
    groups = [[collate(seqs[i + j * batch:i + (j + 1) * batch], n) for j in range(every)]
              for i in range(0, len(seqs) - batch * every + 1, batch * every)]

    def run(gs):
        counted = 0
        for g in gs:
            for data in group_by_length(g) if grouped else g:
                tr.step(data)
                counted += int(counted_length(data[:, 1:]).sum())
        torch.cuda.synchronize()
        return counted
    run(groups[:2] * 3)                                  # eager steps and captures of the lengths seen first
    t0 = time.perf_counter()
    counted = run(groups)
    dt = time.perf_counter() - t0
    return dict(counted_tokens_per_s=round(counted / dt), seconds=round(dt, 3), micro_steps=len(groups) * every,
                graphs=len(tr._graphs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--loop_batches', type=int, default=12)
    args = ap.parse_args()
    kw = CONFIGS['cfg2']['kwargs']
    B, n = CONFIGS['cfg2']['batch'], kw['seq_len']
    res = dict(gpu=gpu_info(torch.cuda.current_device()), config='cfg2', batch=B, steps=args.steps, rounds=args.rounds)
    model = ProGen(**kw, mixed_precision=True)
    params = model.init(0)

    tr = model.trainer(params, cuda_graph=True)
    lengths = list(range(128, n + 1, 128))
    res['lm'], rows = per_length(tr, lambda r, L: tr.step(r, length=L), n, lengths, B, args.steps, args.rounds)
    res['peak_gib'] = dict(cut_384=peak(lambda: [tr.step(rows[384]) for _ in range(2)]),
                           full=peak(lambda: [tr.step(rows[384], length=n) for _ in range(2)]))
    del tr
    torch.cuda.empty_cache()

    ad = model.init_adapters(0, 16)
    tr = model.trainer(params, adapters=ad, cuda_graph=True)
    res['lora_r16'], _ = per_length(tr, lambda r, L: tr.step(r, length=L), n, [384], B, args.steps, args.rounds)
    del tr
    torch.cuda.empty_cache()
    tr = model.trainer(params, adapters=ad, head=model.init_head(0, 3), task='regression', cuda_graph=True)
    y = np.random.default_rng(1).standard_normal((B, 3)).astype(np.float32)
    res['property_r16'], _ = per_length(tr, lambda r, L: tr.property_step(r, y, length=L), n, [384], B, args.steps,
                                        args.rounds)
    del tr, model
    torch.cuda.empty_cache()

    seqs = corpus(16 * 4 * args.loop_batches)
    res['corpus'] = dict(sequences=len(seqs), length='log-normal, median 300, sigma 0.6, clipped to [30, 1000]',
                         median=int(np.median([len(s) for s in seqs])), mean=round(float(np.mean([len(s) for s in seqs])), 1))
    res['loop'] = {f"{'grouped' if g else 'plain'}_{'graph' if c else 'eager'}": loop(kw, params, seqs, g, c)
                   for c in (False, True) for g in (False, True)}
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
