"""Refilled generation (the row queue of the persistent decode kernel) against the static schedule, at the config-5 model.

    python scripts/refill_bench.py [--rounds 3] [--samples 1024]

Model and prompt as scripts/generate_bench.py: d512 L12 n1024 w256 h8 (10 GLU + 2 gMLP layers), ProGen.init(1234), bf16
weights, prompt '[Tax=Mammalia] #', T 1, top_p 0.95.  For batch_size 64 and 8 and three head biases of EOS (as initialised;
raised to about 1 % right after the prompt; banned), `samples` rows are generated twice:
  static: the loop ProGen.generate ran before the queue, kept here: plan_launches + BatchDecoder.generate, one launch of
    batch_size rows after another, each running until its last row ends;
  queue: ProGen.generate, whose slots take the next row when theirs ends.
Reported per case: wall-clock seconds (median), sequences/s, generated tokens/s, and the kernel positions run (prompt
positions included).  The two must give the same tokens; the script checks it.  lock_step_us: device µs per position of
one BatchDecoder.generate launch with EOS banned (every row runs to seq_len) at 8, 12 and 64 rows.  Every measurement is
warmed up once, then all are alternated `rounds` times; medians are reported with the card's name and power limit.
Prints one JSON line."""
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
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from bench import gpu_info                                # noqa: E402
from generate_bench import KW, PROMPT, with_eos_bias      # noqa: E402
from progen_b200 import ProGen                            # noqa: E402
from progen_b200.data import encode_tokens                # noqa: E402
from progen_b200.decode import BatchDecoder               # noqa: E402
from progen_b200.progen import plan_launches              # noqa: E402

SAMPLE = dict(temperature=1.0, top_p=0.95)


def static_generate(dec, rows, batch_size, seed):
    """-> (tokens, generated tokens, positions run) of the static schedule"""
    n = KW['seq_len']
    tokens = np.zeros((len(rows), n), np.int64)
    gen = positions = 0
    for sids, real in plan_launches([len(a) for a in rows], batch_size):
        res = dec.generate([rows[r] for r in sids], sample_ids=sids, seed=seed, **SAMPLE)
        tokens[sids[:real]] = res['ids'][:real]
        ends = np.minimum(res['end'][:real] + 1, n)
        gen += int((ends - res['start'][:real]).sum())
        positions += int(res['start'].min()) - 1 + res['steps_run']
    return tokens, gen, positions


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--samples', type=int, default=1024)
    args = ap.parse_args()
    n = KW['seq_len']
    params = ProGen(**KW).init(1234)
    prime = np.array(encode_tokens(PROMPT), np.int64)
    row = np.zeros(n, np.int64)
    row[1:1 + len(prime)] = prime
    l = ProGen(**KW).apply(params, None, row)[len(prime)].double().cpu().numpy()
    rest = np.log(np.exp(l[1:] - l.max()).sum()) + l.max()
    delta = float(np.log(0.01 / 0.99) + rest - l[0])
    psets = dict(model=params, eos_1pct=with_eos_bias(params, delta), no_eos=with_eos_bias(params, -np.inf))
    models = {k: ProGen(**KW, mixed_precision=True) for k in psets}
    decs = {(k, bs): BatchDecoder(models[k].config, p, batch=bs, weights_dtype=torch.bfloat16)
            for k, p in psets.items() for bs in (64, 8)}
    lock = {B: BatchDecoder(models['no_eos'].config, psets['no_eos'], batch=B, weights_dtype=torch.bfloat16) for B in (8, 12, 64)}
    rows = [prime] * args.samples
    cases = [(k, bs) for bs in (64, 8) for k in psets]
    times = {f'{k}_bs{bs}_{how}': [] for k, bs in cases for how in ('static', 'queue')}
    lock_us = {f'B{B}': [] for B in lock}
    info = {}
    for rnd in range(args.rounds + 1):                          # round 0: warm-up
        for k, bs in cases:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tok_s, gen, positions = static_generate(decs[(k, bs)], rows, bs, seed=rnd)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            q = models[k].generate(psets[k], PROMPT, num_samples=args.samples, batch_size=bs, seed=rnd, **SAMPLE)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if not np.array_equal(q['tokens'], tok_s):
                raise SystemExit(f'{k} batch_size {bs}: the queue and the static schedule gave different tokens')
            if rnd:
                times[f'{k}_bs{bs}_static'].append(t1 - t0)
                times[f'{k}_bs{bs}_queue'].append(t2 - t1)
            if not rnd:                                         # positions of the queue launch (the warm-up's rows again)
                qr = decs[(k, bs)].generate_queue(rows, slots=bs, sample_ids=np.arange(args.samples), seed=rnd, **SAMPLE)
                info[(k, bs)] = dict(generated_tokens=gen, static_positions=positions, queue_positions=qr['steps_run'],
                                     finished=int(q['finished'].sum()))
        for B, dec in lock.items():
            r = dec.generate([prime] * B, seed=rnd, **SAMPLE)
            if rnd:
                lock_us[f'B{B}'].append(r['device_s'] / r['steps_run'] * 1e6)
    out = {}
    for k, bs in cases:
        d = dict(info[(k, bs)])
        for how in ('static', 'queue'):
            v = times[f'{k}_bs{bs}_{how}']
            s = statistics.median(v)
            d[how] = dict(s=s, s_all=v, seqs_per_s=args.samples / s, generated_tokens_per_s=d['generated_tokens'] / s)
        d['speedup'] = d['static']['s'] / d['queue']['s']
        out[f'{k}_bs{bs}'] = d
    print(json.dumps(dict(metric='generation: row queue vs static launches, config-5 model (bf16 weights)', samples=args.samples,
                          rounds=args.rounds, eos_bias_delta=delta, cases=out,
                          lock_step_us={k: dict(median=statistics.median(v), all=v) for k, v in lock_us.items()},
                          gpu=gpu_info(torch.cuda.current_device()))))


if __name__ == '__main__':
    main()
