"""Deep mutational scan of a seeded 300-residue wild type: `ProGen.score` on the explicitly mutated full-length rows
against `ProGen.score_variants` (the scoring forward cut to the counted positions rounded up to 128, DESIGN.md §3.6).

    python scripts/variants_bench.py [--configs cfg2,cfg3w] [--residues 300] [--rounds 3] [--out result.json]

Models (bf16, randomized weights): cfg2 = config 2 (d512, depth 12, h8, w256, n1024, two gMLP layers); cfg3w = the
config-3 width at depth 3 (d1024, h16, w512, n2048: one GLU and two gMLP layers, the stack of the large-config tests).
The 19 x 300 = 5700 single substitutions and the wild type run at batch_size 64 through both routes.  After one warm-up
call of each route, `--rounds` rounds alternate the two routes; each call is timed on the host around work that ends in
a device synchronise, and the median is reported.  Per route: seconds per call, variants/s, token positions computed,
the device memory the call adds (peak allocated minus allocated before the call), and the speed-up.  The two routes must
agree bit for bit (log_likelihood, num_tokens, token_logp, and delta recomputed from the full-length token_logp).  The
card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIGS = {
    'cfg2': dict(num_tokens=256, dim=512, depth=12, heads=8, dim_head=64, seq_len=1024, window_size=256, global_mlp_depth=2),
    'cfg3w': dict(num_tokens=256, dim=1024, depth=3, heads=16, dim_head=64, seq_len=2048, window_size=512, global_mlp_depth=2),
}
AA = 'ACDEFGHIKLMNPQRSTVWY'


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or 'unknown'
    except (OSError, subprocess.TimeoutExpired):
        power = 'unknown'
    return name, power


def timed(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def run(name, residues, rounds, batch_size):
    from oracle import progen_ref as O
    from progen_b200 import ProGen
    from progen_b200.data import collate
    from progen_b200.engine import cut_length
    from progen_b200.variants import scan_sets, variant_rows, parse_mutations
    kw = CONFIGS[name]
    n = kw['seq_len']
    params = O.randomize_params(O.init_params(O.make_config(**kw), 1), 2)
    model = ProGen(**kw, mixed_precision=True)
    wt = ''.join(np.random.default_rng(300).choice(list(AA), size=residues))
    sets, _ = scan_sets(wt, np.arange(1, residues + 1), AA)
    rows = variant_rows(wt, parse_mutations(wt, sets, n), n)            # the wild type, then every variant
    L = cut_length(rows[:, 1:])
    model._ensure_loaded(params)
    full = lambda: model.score(params, rows, batch_size=batch_size, return_tokens=True)
    cut = lambda: model.score_variants(params, wt, sets, batch_size=batch_size, return_tokens=True)
    ref, _, _ = timed(full)                                              # warm-up of both routes
    got, _, _ = timed(cut)
    times, mem = {'full': [], 'cut': []}, {}
    for _ in range(rounds):
        for route, fn in (('full', full), ('cut', cut)):
            _, t, m = timed(fn)
            times[route].append(t)
            mem[route] = max(mem.get(route, 0), m)
    lp = ref['token_logp'].astype(np.float64)
    bitwise = bool(np.array_equal(got['log_likelihood'], ref['log_likelihood'][1:])
                   and np.array_equal(got['num_tokens'], ref['num_tokens'][1:])
                   and np.array_equal(got['token_logp'], ref['token_logp'][1:])
                   and got['wt_log_likelihood'] == ref['log_likelihood'][0]
                   and np.array_equal(got['delta'], (lp[1:] - lp[0]).sum(-1)))
    med = {k: float(np.median(v)) for k, v in times.items()}
    M = len(sets)
    res = dict(config=name, model={k: v for k, v in kw.items() if k != 'num_tokens'}, residues=residues, variants=M,
               rows=M + 1, batch_size=batch_size, cut_length=L, rounds=rounds,
               full=dict(s_per_call=round(med['full'], 3), variants_per_s=round(M / med['full'], 1),
                         tokens_computed=(M + 1) * n, added_memory_gib=round(mem['full'] / 2 ** 30, 3),
                         times_s=[round(t, 3) for t in times['full']]),
               cut=dict(s_per_call=round(med['cut'], 3), variants_per_s=round(M / med['cut'], 1),
                        tokens_computed=(M + 1) * L, added_memory_gib=round(mem['cut'] / 2 ** 30, 3),
                        times_s=[round(t, 3) for t in times['cut']]),
               speedup=round(med['full'] / med['cut'], 2), bitwise_equal=bitwise)
    del model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='cfg2,cfg3w')
    ap.add_argument('--residues', type=int, default=300)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--batch_size', type=int, default=64)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('variants_bench.py needs a CUDA device (an H100)')
    gpu, power = card()
    results = []
    for name in a.configs.split(','):
        r = run(name, a.residues, a.rounds, a.batch_size)
        r.update(gpu=gpu, power_limit=power)
        print(json.dumps(r), flush=True)
        results.append(r)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(results, f, indent=1)
    if not all(r['bitwise_equal'] for r in results):
        sys.exit('score_variants and score differ')


if __name__ == '__main__':
    main()
