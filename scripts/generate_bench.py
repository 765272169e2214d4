"""Cost of the standard sampler (sampler 1), of its constraints, and gain of the EOS early exit, at the config-5 model.

    python scripts/generate_bench.py [--rounds 3] [--samples 256] [--skip_end_to_end]

Model: d512 L12 n1024 w256 h8 (10 GLU + 2 gMLP layers), seeded parameters (ProGen.init(1234), as bench.py --config cfg5),
bf16 weights in the persistent decode kernel; prompt '[Tax=Mammalia] #'.
  per_position: device time of one launch (CUDA events) over the positions it ran, at B = 1, 8, 12, 64 sequences, for
    the reference sampler (BatchDecoder.sample, top_k 25, Gumbel noise: what bench.py --config cfg5 runs) and for sampler 1
    (BatchDecoder.generate, T 1, top_p 0.95; positions = steps_run, so an early exit is accounted for).  Sampler 1 plans
    the attention and SGU work splits for 1, 8 or 64 rows (the largest launch of the batch tile's class); B = 12 shows
    what that costs a launch smaller than its class's largest.  `con` is sampler 1 with the constraints a protein user
    sets: the 20 amino acids as the alphabet (a logit bias banning every other id but EOS), min_new_tokens 64,
    repetition_penalty 1.2 over a 16-position window, against `std_full`, sampler 1 without them.  Both run with EOS
    unreachable (the `no_eos` head bias below), so both consume every position: a position's cost grows with its index
    (the gMLP layers' causal history sum), and the alphabet makes EOS so likely that a constrained launch would
    otherwise stop after about a tenth of the positions of a plain one.  `pos` is sampler 1 with a full-length position
    table (`position_bias`, one [seq_len, V] table for every row): a random finite profile over the 20 amino acids
    (every other id but EOS at -inf) with a fixed residue (a one-hot row) every 50 positions, against `std_full` too.
  end_to_end: wall clock of ProGen.generate(num_samples=`samples`, batch_size=64, T 1, top_p 0.95) including the host
    copies, for three parameter sets: as initialised (`model`), the head bias of token 0 raised so that EOS has probability
    about 1 % right after the prompt (`eos_1pct`), and EOS made unreachable by a -inf head bias (`no_eos`: every sequence
    runs to seq_len, the run without the early exit).
Every measurement is warmed up once, then all of them are alternated `rounds` times; medians are reported with the card's
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
from generate import alphabet_bias                        # noqa: E402
from progen_b200 import ProGen                            # noqa: E402
from progen_b200.data import encode_tokens                # noqa: E402
from progen_b200.decode import BatchDecoder               # noqa: E402
from progen_b200.engine import P                          # noqa: E402

KW = dict(num_tokens=256, dim=512, seq_len=1024, depth=12, heads=8, dim_head=64, window_size=256, global_mlp_depth=2,
          ff_glu=True)
PROMPT = '[Tax=Mammalia] #'
CONSTRAINED = dict(logit_bias=alphabet_bias('ACDEFGHIKLMNPQRSTVWY', KW['num_tokens']), min_new_tokens=64,
                   repetition_penalty=1.2, repetition_window=16)


def with_eos_bias(params, delta):
    out = {k: dict(v) for k, v in params.items()}
    b = np.array(params[P + 'linear']['b'], np.float32, copy=True)
    b[0] = delta if np.isinf(delta) else b[0] + delta
    out[P + 'linear'] = {**params[P + 'linear'], 'b': b}
    return out


def position_table(n, V, seed=7):
    """[1, n, V]: a random finite profile over the 20 amino acids at every generated offset, EOS left at 0, and every
    50th offset a fixed residue (0 at one amino acid, -inf everywhere else)"""
    rng = np.random.default_rng(seed)
    aa = np.array(encode_tokens('ACDEFGHIKLMNPQRSTVWY'), np.int64)
    t = np.full((n, V), -np.inf, np.float32)
    t[:, 0] = 0.0
    t[:, aa] = rng.normal(0.0, 1.0, (n, len(aa))).astype(np.float32)
    for j in range(49, n, 50):
        t[j] = -np.inf
        t[j, rng.choice(aa)] = 0.0
    return t[None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--samples', type=int, default=256)
    ap.add_argument('--skip_end_to_end', action='store_true', help='per-position launches only')
    args = ap.parse_args()
    n = KW['seq_len']
    params = ProGen(**KW).init(1234)
    prime = np.array(encode_tokens(PROMPT), np.int64)
    # EOS about 1 % likely right after the prompt: shift the head bias of token 0 by the log-odds it needs there
    row = np.zeros(n, np.int64)
    row[1:1 + len(prime)] = prime
    l = ProGen(**KW).apply(params, None, row)[len(prime)].double().cpu().numpy()
    rest = np.log(np.exp(l[1:] - l.max()).sum()) + l.max()
    delta = float(np.log(0.01 / 0.99) + rest - l[0])
    psets = dict(model=params, eos_1pct=with_eos_bias(params, delta), no_eos=with_eos_bias(params, -np.inf))
    models = {k: ProGen(**KW, mixed_precision=True) for k in psets}
    decs = {B: BatchDecoder(models['model'].config, params, batch=B, weights_dtype=torch.bfloat16) for B in (1, 8, 12, 64)}
    full = {B: BatchDecoder(models['model'].config, psets['no_eos'], batch=B, weights_dtype=torch.bfloat16) for B in decs}

    def quirk(B, seed):
        _, _, secs = decs[B].sample([prime] * B if B > 1 else prime, top_k=25, add_bos=True, greedy=False, seed=seed)
        return secs / (n - 1 - (len(prime) - 1))                # positions first .. n-2 of the timed launch

    def std(B, seed, dec=decs, **cons):
        r = dec[B].generate([prime] * B, temperature=1.0, top_p=0.95, seed=seed, **cons)
        return r['device_s'] / r['steps_run']

    def e2e(name, seed):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = models[name].generate(psets[name], PROMPT, num_samples=args.samples, temperature=1.0, top_p=0.95, seed=seed,
                                  batch_size=64)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, int(r['length'].sum()), int(r['finished'].sum())

    table = position_table(n, KW['num_tokens'])
    per_pos = {f'{s}_B{B}': [] for B in decs for s in ('quirk', 'std', 'std_full', 'con', 'pos')}
    ends = {k: [] for k in psets}
    for rnd in range(args.rounds + 1):                          # round 0: warm-up
        for B in decs:
            q, s = quirk(B, 100 + rnd), std(B, 100 + rnd)
            f, c = std(B, 100 + rnd, full), std(B, 100 + rnd, full, **CONSTRAINED)
            pt = std(B, 100 + rnd, full, position_bias=(table, np.zeros(B, np.int64)))
            if rnd:
                per_pos[f'quirk_B{B}'].append(q)
                per_pos[f'std_B{B}'].append(s)
                per_pos[f'std_full_B{B}'].append(f)
                per_pos[f'con_B{B}'].append(c)
                per_pos[f'pos_B{B}'].append(pt)
        for name in ([] if args.skip_end_to_end else psets):
            r = e2e(name, rnd)
            if rnd:
                ends[name].append(r)
    res = dict(per_position_us={k: dict(median=statistics.median(v) * 1e6, all=[x * 1e6 for x in v]) for k, v in per_pos.items()})
    res['std_over_quirk'] = {f'B{B}': statistics.median(per_pos[f'std_B{B}']) / statistics.median(per_pos[f'quirk_B{B}'])
                             for B in decs}
    res['con_over_std'] = {f'B{B}': statistics.median(per_pos[f'con_B{B}']) / statistics.median(per_pos[f'std_full_B{B}'])
                           for B in decs}
    res['pos_over_std'] = {f'B{B}': statistics.median(per_pos[f'pos_B{B}']) / statistics.median(per_pos[f'std_full_B{B}'])
                           for B in decs}
    e = {}
    for name, v in ends.items():
        if not v:
            continue
        secs = statistics.median([x[0] for x in v])
        tok = v[0][1]
        e[name] = dict(s=secs, s_all=[x[0] for x in v], seqs_per_s=args.samples / secs, generated_tokens=tok,
                       generated_tokens_per_s=tok / secs, finished=v[0][2])
    res['end_to_end'] = e
    if e:
        res['early_exit_speedup_eos_1pct'] = e['no_eos']['s'] / e['eos_1pct']['s']
    print(json.dumps(dict(metric='generation: sampler-1 and constraint cost per position and EOS early exit, config-5 model (bf16 weights)',
                          samples=args.samples, rounds=args.rounds, eos_bias_delta=delta, **res,
                          gpu=gpu_info(torch.cuda.current_device()))))


if __name__ == '__main__':
    main()
