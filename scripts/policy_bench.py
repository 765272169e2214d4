"""Policy-gradient fine-tuning (DESIGN.md §3.14): where one design.py iteration spends its device time.

    python scripts/policy_bench.py [--iterations 3] [--reps 20]

Config 2 (bf16), ProGen.init(0) as the base, adapters of rank 16 trained on it, the reference a second config-2 model
on the base, the reward model a third one with a random one-output head; 8 prompts x 8 samples per iteration,
max_length 512, temperature 1, beta 0.04, one policy step over the 64 rows.  Reported, medians over `iterations`
iterations after one warm-up iteration, each part timed with CUDA events and a synchronise:
  refresh_ms: BatchDecoder.load_weights from the trainer's adapters (progen_decode_load_weight on the 4 adapted
    projections of every layer);
  generate_ms: Trainer.generate of the 64 rows; reward_ms: ProGen.predict of the reward model on them;
  step_ms: Trainer.policy_step (the reference's forward, the policy's forward, the head, the backward and AdamW) at the
    rows' cut length;
  head_ms: progen_policy_head alone at that length, against its HBM floor T V (4 + 4 + 2) bytes / 3.35 TB/s (policy and
    reference logits in fp32, bf16 dlogits; the data-sheet bandwidth of the H100 SXM);
  refresh_kernel_ms: the refresh alone, against its floor: every adapted W read in fp32 and written in bf16, plus A and B.
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
from progen_b200.lora import adapter_modules             # noqa: E402
from progen_b200.policy import group_advantages, samples_to_rows   # noqa: E402

HBM_BYTES_PER_S = 3.35e12
PROMPTS = ['M' + c for c in 'KTAYIAKQ']
SAMPLES, MAX_LENGTH, RANK, BETA = 8, 512, 16, 0.04


def timed(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iterations', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    kw = CONFIGS['cfg2']['kwargs']
    model, ref, scorer = (ProGen(**kw, mixed_precision=True) for _ in range(3))
    params = model.init(0)
    head = scorer.init_head(1, 1)
    tr = model.trainer(params, adapters=model.init_adapters(2, RANK), learning_rate=1e-5, grad_accum_every=1,
                       data_parallel=False, reference=ref, reference_params=params)
    parts = dict(refresh=[], generate=[], reward=[], step=[])
    for it in range(args.iterations + 1):
        t_refresh, dec = timed(lambda: tr._generate_decoder(SAMPLES * len(PROMPTS)))
        t_gen, s = timed(lambda: tr.generate(PROMPTS, num_samples=SAMPLES, max_length=MAX_LENGTH, seed=it))
        rows, span = samples_to_rows(s)
        t_rew, pred = timed(lambda: scorer.predict(params, head, rows)['prediction'])
        adv = group_advantages(pred[:, 0], SAMPLES)
        t_step, _ = timed(lambda: tr.policy_step(rows, span, adv, BETA))
        if it:
            for k, t in zip(parts, (t_refresh, t_gen, t_rew, t_step)):
                parts[k].append(t)
    eng, lo = tr.eng, tr.lora
    n = eng.row_length(rows)
    B = eng.load_policy(rows, span, adv.astype(np.float32), n, reference=True)
    a = eng.acts.view(B, n)
    te = eng.teacher
    ta = te.infer.view(B, teacher_length(n, te.n))
    te._forward_device(ta)
    eng._forward_device(a)
    lib, st = L.load(), L.stream()

    def head_launch():
        L.check(lib.progen_policy_head(a.logits.data_ptr(), L.F32, ta.logits.data_ptr(), ta.n, a.labels.data_ptr(),
                                       eng.pol['span'].data_ptr(), eng.pol['adv'].data_ptr(),
                                       eng.pol['scratch'].data_ptr(), eng.pol['stats'].data_ptr(), eng.loss.data_ptr(),
                                       a.grad['dlogits'].data_ptr(), eng.act_dt, B, n, eng.V, BETA, 1.0 / B, st),
                'policy_head')
    head_ms = statistics.median(timed(head_launch, args.reps)[0] for _ in range(3))
    head_floor = B * n * eng.V * (4 + 4 + 2) / HBM_BYTES_PER_S * 1e3
    refresh_ms = statistics.median(timed(lambda: dec.load_weights(eng, lo), args.reps)[0] for _ in range(3))
    elems = sum(i * o for _, i, o, _ in adapter_modules(model.config))
    ab = sum(RANK * (i + o) for _, i, o, _ in adapter_modules(model.config))
    refresh_floor = (elems * (4 + 2) + ab * 4) / HBM_BYTES_PER_S * 1e3
    med = {k: round(statistics.median(v), 3) for k, v in parts.items()}
    out = dict(gpu=gpu_info(torch.cuda.current_device()), config='cfg2', dtype='bf16', lora_rank=RANK,
               prompts=len(PROMPTS), samples_per_prompt=SAMPLES, max_length=MAX_LENGTH, beta=BETA,
               iterations=args.iterations, step_length=int(n), mean_generated=float(s['length'].mean()),
               iteration_ms=dict(med, total=round(sum(med.values()), 3)),
               head_ms=round(head_ms, 4), head_floor_ms=round(head_floor, 4), head_over_floor=round(head_ms / head_floor, 2),
               refresh_kernel_ms=round(refresh_ms, 4), refresh_floor_ms=round(refresh_floor, 4),
               refresh_over_floor=round(refresh_ms / refresh_floor, 2))
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
