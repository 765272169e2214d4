"""Cost of preference (DPO) fine-tuning at the config-2 shape: the captured preference step against the captured plain
training step of the same rows, and the preference head alone against the cross-entropy head it replaces.

    python scripts/dpo_bench.py [--pairs 32] [--steps 10] [--rounds 3]

Model: d512 L12 n1024 w256 h8, 10 GLU + 2 gMLP layers, bf16 engine, ProGen.init(0).  Input: 2 * pairs uniform-random
rows from seed 42 (data.synthetic_iterator, the training benchmark's distribution; 32 pairs = the benchmark's 64 rows),
chosen = the first half, with reference log-likelihoods = `score` at the same parameters plus N(0, 3) noise.  Both steps
run on one Trainer, each captured into its own CUDA graph (forward, head, backward, clip, AdamW); a round times `steps`
replays of one graph, then of the other, between CUDA events, and the median over `rounds` alternated rounds is
reported.  The heads are timed alone on the logits of one forward, 50 launches between CUDA events.  Prints one JSON line
with the card name and power limit."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_info                               # noqa: E402
from progen_b200 import ProGen, lib as L                 # noqa: E402
from progen_b200.data import synthetic_iterator          # noqa: E402

KW = dict(num_tokens=256, dim=512, seq_len=1024, depth=12, heads=8, dim_head=64, window_size=256, global_mlp_depth=2,
          ff_glu=True)


def timed(fn, n):
    """ms per call of fn over n calls, between CUDA events"""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=32)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    P, B = args.pairs, 2 * args.pairs
    model = ProGen(**KW, mixed_precision=True)
    params = model.init(0)
    rows = next(synthetic_iterator(KW['seq_len'], B, seed=42))
    ref = model.score(params, rows)['log_likelihood'] + np.random.default_rng(0).normal(0, 3, B).astype(np.float32)
    c, r, rc, rr = rows[:P], rows[P:], ref[:P], ref[P:]
    tr = model.trainer(params, learning_rate=1e-6, grad_accum_every=1)
    eng = tr.eng
    beta = 0.1
    # two eager steps of each kind, then one graph each
    for _ in range(2):
        tr.step(rows)
        tr.preference_step(c, r, rc, rr, beta=beta)
    torch.cuda.synchronize()
    g_plain = tr.capture_graph(B, B, install=False)
    g_pref = tr._capture(B, None, lambda: eng.preference_step_device(P, beta, P), install=False)
    eng.load_preference(*(np.concatenate(x) for x in ((c, r), (rc, rr))))
    for g in (g_plain, g_pref):
        timed(g.replay, 2)
    plain, pref = [], []
    for _ in range(args.rounds):
        plain.append(timed(g_plain.replay, args.steps))
        pref.append(timed(g_pref.replay, args.steps))
    # the heads alone, on the logits of one forward
    eng._forward_device()
    st = L.stream()
    ce = lambda: L.check(eng.lib.progen_ce_fwd_bwd(eng.logits.data_ptr(), L.F32, eng.labels.data_ptr(), eng.ce_w.data_ptr(),
                                                   eng.loss.data_ptr(), eng.dlogits.data_ptr(), eng.act_dt, B, eng.n, eng.V,
                                                   1.0 / B, st), 'ce_fwd_bwd')
    head = lambda: L.check(eng.lib.progen_preference_head(
        eng.logits.data_ptr(), L.F32, eng.labels.data_ptr(), eng.ref.data_ptr(), eng.logp.data_ptr(), eng.seq_ll.data_ptr(),
        eng.seq_count.data_ptr(), eng.ce_w.data_ptr(), eng.stats.data_ptr(), eng.loss.data_ptr(), eng.ce_scratch.data_ptr(),
        eng.dlogits.data_ptr(), eng.act_dt, P, eng.n, eng.V, beta, 1.0 / P, st), 'preference_head')
    for f in (ce, head):
        timed(f, 5)
    ce_ms, head_ms = [], []
    for _ in range(args.rounds):
        ce_ms.append(timed(ce, 50))
        head_ms.append(timed(head, 50))
    mp, mq = statistics.median(plain), statistics.median(pref)
    logits_mib = eng.logits.numel() * 4 / 2 ** 20
    print(json.dumps(dict(
        gpu=gpu_info(torch.cuda.current_device()), pairs=P, rows=B, seq_len=KW['seq_len'],
        plain_step_ms=round(mp, 3), preference_step_ms=round(mq, 3), preference_over_plain=round(mq / mp, 4),
        plain_rounds_ms=[round(x, 3) for x in plain], preference_rounds_ms=[round(x, 3) for x in pref],
        ce_head_ms=round(statistics.median(ce_ms), 4), preference_head_ms=round(statistics.median(head_ms), 4),
        preference_head_share_of_step=round(statistics.median(head_ms) / mq, 5), fp32_logits_mib=round(logits_mib, 1))),
        flush=True)


if __name__ == '__main__':
    main()
