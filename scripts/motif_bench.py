"""Cost of the motif constraints (`generate(require=, avoid=)`) in the standard sampler, at the config-5 model.

    python scripts/motif_bench.py [--rounds 3]

Model: d512 L12 n1024 w256 h8 (10 GLU + 2 gMLP layers), seeded parameters (ProGen.init(1234), as bench.py --config cfg5),
bf16 weights in the persistent decode kernel, prompt '[Tax=Mammalia] #', EOS unreachable (a -inf head bias), so every
launch consumes every position.  per_position_us: device time of one BatchDecoder.generate launch (CUDA events) over its
steps_run, at B = 1, 8 and 64 rows, for sampler 1 alone (T 1, top_p 0.95: `std`) and with one required pattern, the C2H2
zinc finger (PS00028), and two avoided ones, N-glycosylation sites and a tryptophan pair (`motif`).  Each draw then runs
the motif step for its <= 2 ids per thread over 3 patterns of 64-bit operations, next to the filter's O(V^2) rank counts.
Every measurement is warmed up once, then the two are alternated `rounds` times; medians are reported with the card's
name and power limit.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_info                                # noqa: E402
from progen_b200 import ProGen                            # noqa: E402
from progen_b200.data import encode_tokens                # noqa: E402
from progen_b200.decode import BatchDecoder               # noqa: E402
from progen_b200.motif import Motif                       # noqa: E402
from generate_bench import KW, PROMPT, with_eos_bias      # noqa: E402

REQUIRE = 'C-x(2,4)-C-x(3)-[LIVMFYWC]-x(8)-H-x(3,5)-H'
AVOID = ['N-{P}-[ST]-{P}', 'W-W']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    params = with_eos_bias(ProGen(**KW).init(1234), -np.inf)
    prime = np.array(encode_tokens(PROMPT), np.int64)
    cfg = ProGen(**KW).config
    motif = Motif(REQUIRE, AVOID, KW['num_tokens'])
    decs = {B: BatchDecoder(cfg, params, batch=B, weights_dtype=torch.bfloat16) for B in (1, 8, 64)}

    def run(B, seed, **kw):
        r = decs[B].generate([prime] * B, temperature=1.0, top_p=0.95, seed=seed, **kw)
        return r['device_s'] / r['steps_run'], r

    per_pos = {f'{s}_B{B}': [] for B in decs for s in ('std', 'motif')}
    matched = {}
    for rnd in range(args.rounds + 1):                          # round 0: warm-up
        for B in decs:
            s, _ = run(B, 100 + rnd)
            m, r = run(B, 100 + rnd, motif=motif)
            if rnd:
                per_pos[f'std_B{B}'].append(s)
                per_pos[f'motif_B{B}'].append(m)
                gen = [r['ids'][b, r['start'][b]:] for b in range(B)]
                matched[f'B{B}'] = float(motif.matches(gen).mean())
    res = dict(per_position_us={k: dict(median=statistics.median(v) * 1e6, all=[x * 1e6 for x in v]) for k, v in per_pos.items()})
    res['motif_over_std'] = {f'B{B}': statistics.median(per_pos[f'motif_B{B}']) / statistics.median(per_pos[f'std_B{B}'])
                             for B in decs}
    res['rows_matching'] = matched
    print(json.dumps(dict(metric='generation: motif constraint cost per position, config-5 model (bf16 weights)',
                          require=REQUIRE, avoid=AVOID, rounds=args.rounds, **res, gpu=gpu_info(torch.cuda.current_device()))))


if __name__ == '__main__':
    main()
