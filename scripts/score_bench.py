"""Throughput and memory of sequence scoring (ProGen.score) at the config-2 shape, against the route available without
it: `.apply` (the training forward, which allocates every buffer the backward pass needs) followed by a torch
log_softmax / gather / Q8 mask.

    python scripts/score_bench.py [--rows 1024] [--rounds 3]

Model: d512 L12 n1024 w256 h8, 10 GLU + 2 gMLP layers, bf16 engine, seeded random parameters (ProGen.init(0)).  Input:
`rows` uniform-random rows from seed 42 (data.synthetic_iterator, the training benchmark's distribution).  Each timed
sample is one whole call over all rows (H2D copies, forwards, scoring kernels, D2H copies), between CUDA events on the
current stream followed by a synchronise; the three paths are warmed up once, then alternated `rounds` times and the
median is reported.  Memory: torch.cuda.max_memory_allocated during a path's first call minus what was allocated
before it (the buffers the path allocates plus its transients), and the absolute peak.  `e2e_share_of_989` is the
end-to-end forward FLOP rate (bench.fwd_flops_per_token x tokens/s) over the H100 SXM data-sheet dense BF16 rate; it is
not a kernel's share of peak.  Prints one JSON line."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import fwd_flops_per_token, gpu_info          # noqa: E402
from progen_b200 import ProGen                           # noqa: E402
from progen_b200.data import synthetic_iterator          # noqa: E402

KW = dict(num_tokens=256, dim=512, seq_len=1024, depth=12, heads=8, dim_head=64, window_size=256, global_mlp_depth=2,
          ff_glu=True)
PEAK_TFLOPS = 989.0        # NVIDIA H100 SXM data sheet, dense BF16, 700 W


def apply_route(model, params, rows, batch):
    """per-sequence log-likelihood the way it is written without ProGen.score"""
    V = model.config['num_tokens']
    out = []
    for r0 in range(0, rows.shape[0], batch):
        chunk = rows[r0:r0 + batch]
        logits = model.apply(params, None, chunk[:, :-1])
        labels = torch.as_tensor(chunk[:, 1:].astype(np.int64)).cuda()
        lp = torch.log_softmax(logits, -1).gather(-1, labels.clamp(0, V - 1)[..., None])[..., 0]
        pad = labels == 0
        mask = ~pad | ((pad.cumsum(-1) == 1) & pad)
        out.append((lp * mask).sum(-1).cpu())
    return torch.cat(out).numpy()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    res = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=1024)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    n = KW['seq_len']
    rows = next(synthetic_iterator(n, args.rows, seed=42))
    params = ProGen(**KW).init(0)
    # one model (engine) per path, so that each path's activation buffers are its own
    paths = {'score_b64': (ProGen(**KW, mixed_precision=True), lambda m: m.score(params, rows, batch_size=64)['log_likelihood']),
             'score_b256': (ProGen(**KW, mixed_precision=True), lambda m: m.score(params, rows, batch_size=256)['log_likelihood']),
             'apply_b64': (ProGen(**KW, mixed_precision=True), lambda m: apply_route(m, params, rows, 64))}
    per_pass = dict(score_b64=64, score_b256=256, apply_b64=64)      # sequences per forward pass
    mem, ll = {}, {}
    for name, (model, fn) in paths.items():                      # first call: warm-up and footprint
        model._ensure_loaded(params)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ll[name] = fn(model)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        tokens_per_pass = min(args.rows, per_pass[name]) * n
        mem[name] = dict(added_gib=(peak - base) / 2**30, added_kib_per_token=(peak - base) / tokens_per_pass / 1024,
                         peak_gib=peak / 2**30)
    times = {k: [] for k in paths}
    for _ in range(args.rounds):                                 # alternated in the same process
        for name, (model, fn) in paths.items():
            t, _ = timed(lambda: fn(model))
            times[name].append(t)
    F = fwd_flops_per_token(KW)
    tok = args.rows * n
    res = {}
    for name in paths:
        t = statistics.median(times[name])
        res[name] = dict(s=t, s_all=times[name], tokens_per_s=tok / t, seqs_per_s=args.rows / t,
                         e2e_tflops=F * tok / t / 1e12, e2e_share_of_989=F * tok / t / 1e12 / PEAK_TFLOPS, **mem[name])
    print(json.dumps(dict(metric='ProGen.score throughput, config-2 shape (d512 L12 n1024 w256 h8, bf16), %d rows' % args.rows,
                          rows=args.rows, seq_len=n, rounds=args.rounds, fwd_flops_per_token=F, peak_tflops_datasheet=PEAK_TFLOPS,
                          paths=res, speedup_b64_vs_apply=res['apply_b64']['s'] / res['score_b64']['s'],
                          ll_max_abs_diff_b64_vs_b256=float(np.abs(ll['score_b64'] - ll['score_b256']).max()),
                          ll_max_abs_diff_score_vs_apply=float(np.abs(ll['score_b64'] - ll['apply_b64']).max()),
                          mean_ll_per_row=float(np.mean(ll['score_b64'])), gpu=gpu_info(torch.cuda.current_device()))))


if __name__ == '__main__':
    main()
