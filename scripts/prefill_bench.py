"""Prompt prefill of generation: the decode kernel walking the prompt one position at a time (prefill='decode') against one
inference forward plus the cache scatter (prefill='forward'), at the config-5 model.

    python scripts/prefill_bench.py [--rounds 3] [--lengths 17,128,512,896] [--rows 1,8,64]

Model: d512 L12 n1024 w256 h8 (10 GLU + 2 gMLP layers), seeded parameters (ProGen.init(1234), as bench.py --config cfg5),
mixed precision: bf16 weights in the decode kernel, the tensor-core forward.  One random prompt of each length, `rows`
samples of it per launch (num_samples = batch_size = rows).
  prefill_ms: device time of the prefill alone.  'decode': CUDA events around the kernel launch over positions 0 .. P-1
    (BatchDecoder.generate's prefill_s); 'forward': events around BatchDecoder.prefill (the forward over the one distinct
    prompt and the scatter into the caches of every row).
  generate_s: wall clock of the whole ProGen.generate call (T 1, top_p 0.95, host copies included) with EOS made
    unreachable (a -inf head bias), so every row runs to seq_len in both modes and the two do the same decode work after
    the prompt.
  first_draw_max_abs_dlogit: max |logit difference| between the modes at the first drawn position, over the rows.
Every measurement is warmed up once, then the modes are alternated `rounds` times; medians are reported with the card's
name and power limit.  Prints one JSON line."""
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

from bench import gpu_info                                # noqa: E402
from progen_b200 import ProGen                            # noqa: E402
from progen_b200.decode import BatchDecoder               # noqa: E402
from progen_b200.engine import P as PREFIX                # noqa: E402

KW = dict(num_tokens=256, dim=512, seq_len=1024, depth=12, heads=8, dim_head=64, window_size=256, global_mlp_depth=2,
          ff_glu=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--lengths', default='17,128,512,896')
    ap.add_argument('--rows', default='1,8,64')
    args = ap.parse_args()
    lengths = [int(x) for x in args.lengths.split(',')]
    rows = [int(x) for x in args.rows.split(',')]
    params = ProGen(**KW).init(1234)
    no_eos = {k: dict(v) for k, v in params.items()}
    b = np.array(params[PREFIX + 'linear']['b'], np.float32, copy=True)
    b[0] = -np.inf
    no_eos[PREFIX + 'linear'] = {**params[PREFIX + 'linear'], 'b': b}
    model = ProGen(**KW, mixed_precision=True)
    model._ensure_loaded(params)
    rng = np.random.default_rng(5)
    prompts = {L: rng.integers(1, 256, L).astype(np.int64) for L in lengths}
    decs = {B: BatchDecoder(model.config, params, batch=B, weights_dtype=torch.bfloat16) for B in rows}
    gen_kw = dict(temperature=1.0, top_p=0.95)

    def prefill_decode(L, B, seed):
        r = decs[B].generate([prompts[L]] * B, seed=seed, max_length=L + 2, **gen_kw)
        return r['prefill_s']

    def prefill_forward(L, B, seed):
        dec = decs[B]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        P = dec.prefill(model.engine, [prompts[L]] * B)
        e1.record()
        dec.generate([prompts[L]] * B, seed=seed, max_length=L + 2, prefilled=P, **gen_kw)
        return e0.elapsed_time(e1) / 1e3

    def whole(L, B, mode, seed):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.generate(no_eos, [prompts[L]], num_samples=B, batch_size=B, seed=seed, prefill=mode, **gen_kw)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    # first-draw logits of both modes
    dlogit = {}
    for B in rows:
        ka = BatchDecoder(model.config, params, batch=B, weights_dtype=torch.bfloat16, keep_logits=True)
        for L in lengths:
            ka.generate([prompts[L]] * B, temperature=0.0, max_length=L + 2)
            la = ka.logits_all[:B, L].clone()
            P = ka.prefill(model.engine, [prompts[L]] * B)
            ka.generate([prompts[L]] * B, temperature=0.0, max_length=L + 2, prefilled=P)
            dlogit[f'L{L}_B{B}'] = float((ka.logits_all[:B, L] - la).abs().max())
        del ka
        torch.cuda.empty_cache()

    keys = [(L, B) for L in lengths for B in rows]
    t = {f'{m}_L{L}_B{B}': [] for L, B in keys for m in ('prefill_decode', 'prefill_forward', 'generate_decode', 'generate_forward')}
    for rnd in range(args.rounds + 1):                          # round 0: warm-up
        for L, B in keys:
            got = dict(prefill_decode=prefill_decode(L, B, rnd), prefill_forward=prefill_forward(L, B, rnd),
                       generate_decode=whole(L, B, 'decode', rnd), generate_forward=whole(L, B, 'forward', rnd))
            if rnd:
                for m, v in got.items():
                    t[f'{m}_L{L}_B{B}'].append(v)
    med = {k: statistics.median(v) for k, v in t.items()}
    table = {}
    for L, B in keys:
        k = f'L{L}_B{B}'
        table[k] = dict(prefill_ms=dict(decode=med[f'prefill_decode_{k}'] * 1e3, forward=med[f'prefill_forward_{k}'] * 1e3,
                                        speedup=med[f'prefill_decode_{k}'] / med[f'prefill_forward_{k}']),
                        generate_s=dict(decode=med[f'generate_decode_{k}'], forward=med[f'generate_forward_{k}'],
                                        speedup=med[f'generate_decode_{k}'] / med[f'generate_forward_{k}']),
                        first_draw_max_abs_dlogit=dlogit[k])
    print(json.dumps(dict(metric="generation prefill: prefill='decode' vs 'forward', config-5 model (mixed precision)",
                          rounds=args.rounds, results=table, all={k: v for k, v in t.items()},
                          gpu=gpu_info(torch.cuda.current_device()))))


if __name__ == '__main__':
    main()
