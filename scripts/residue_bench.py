"""Cost of a per-residue fine-tuning step (the property head at every position, rank-r adapters, frozen base) against the
property step (the head on the pooled embedding) on the same rows, and the residue head's kernels against their HBM floor.

    python scripts/residue_bench.py [--rank 16] [--steps 10] [--rounds 3] [--skip_cfg4]

Steps: config 2 (batch 64) at row length 384 and at seq_len, config 4 (batch 4) at seq_len.  One trainer per mode on
ProGen.init(0), the same adapters (rank r, seed 0) and the same uniform-random rows (seed 42, data.synthetic_iterator),
cut to their first 383 residues for the 384 case; the residue head is a 3-class classification head with a random class
at every residue, the property head a 3-class head with a random class per row.  Each step is captured into a CUDA graph
after two eager steps; a round times `steps` replays between CUDA events, and the median over `rounds` rounds is
reported.  The two modes' rounds alternate when both trainers fit on the device together; otherwise each mode is timed
while it is the only one resident.

Kernels: progen_residue_head (training: count, head, loss) and progen_residue_head_wgrad at the config-2 shape (64 x 1024
positions, d 512, bf16 h, 3 classes, every residue labelled), each timed with CUDA events over 50 launches, against the
HBM floor of the bytes the shapes imply: h read twice (head, wgrad) and dy written once, in bf16, over 3.35 TB/s.
Prints one JSON line with the card name and power limit."""
import argparse
import gc
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, gpu_info                      # noqa: E402
from progen_b200 import ProGen, lib as L                 # noqa: E402
from progen_b200.data import synthetic_iterator          # noqa: E402
from progen_b200.property import residue_positions       # noqa: E402

HBM_BYTES_PER_S = 3.35e12                                # H100 SXM data sheet


def make(kw, params, rows, targets, rank, mode, length):
    """a trainer of one mode with its step captured at `length` -> replay function"""
    model = ProGen(**kw, mixed_precision=True)
    tr = model.trainer(params, adapters=model.init_adapters(0, rank), head=model.init_head(0, 3), task='classification',
                       cuda_graph=True)
    step = tr.residue_step if mode == 'residue' else tr.property_step
    for _ in range(3):                                    # two eager steps, the capture, then one replay
        step(rows, targets, length=length)
    assert tr._graph is not None and tr._graph_length == length
    torch.cuda.synchronize()
    return tr._replay, tr


def timed_round(replay, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def free():
    gc.collect()
    torch.cuda.empty_cache()


def steps_case(name, kw, batch, length, rank, steps, rounds):
    n = kw['seq_len']
    params = ProGen(**kw).init(0)
    rows = next(synthetic_iterator(n, batch, seed=42)).astype(np.int32)
    rows[:, 1:][rows[:, 1:] == 0] = 1                     # no pad inside a row: every position up to the cut holds a residue
    if length < n:
        rows[:, length:] = 0
    rng = np.random.default_rng(0)
    res_t = np.where(residue_positions(rows), rng.integers(0, 3, (batch, n)), -1)
    prop_t = rng.integers(0, 3, batch)
    rr = tr_r = rp = tr_p = None
    try:
        rr, tr_r = make(kw, params, rows, res_t, rank, 'residue', length)
        try:
            rp, tr_p = make(kw, params, rows, prop_t, rank, 'property', length)
        except torch.cuda.OutOfMemoryError:
            rp = tr_p = None
        alternated = rp is not None
        tres, tprop = [], []
        if alternated:
            for _ in range(rounds):
                tres.append(timed_round(rr, steps))
                tprop.append(timed_round(rp, steps))
        else:                                             # the two trainers do not fit together: each mode alone
            free()
            tres = [timed_round(rr, steps) for _ in range(rounds)]
            res_loss = float(tr_r.eng.loss.item())
            rr = tr_r = None
            free()
            rp, tr_p = make(kw, params, rows, prop_t, rank, 'property', length)
            tprop = [timed_round(rp, steps) for _ in range(rounds)]
        out = dict(config=name, batch=batch, length=length, rank=rank, alternated=alternated,
                   residue_step_ms=statistics.median(tres), residue_step_ms_rounds=tres,
                   property_step_ms=statistics.median(tprop), property_step_ms_rounds=tprop,
                   residue_loss=float(tr_r.eng.loss.item()) if tr_r is not None else res_loss,
                   labelled_positions=int((res_t >= 0).sum()))
        out['residue_over_property'] = out['residue_step_ms'] / out['property_step_ms']
        return out
    except (torch.cuda.OutOfMemoryError, L.ProgenError) as e:
        return dict(config=name, batch=batch, length=length, error=f'{type(e).__name__}: {str(e)[:200]}')
    finally:
        rr = tr_r = rp = tr_p = None
        free()


def kernels(B=64, n=1024, d=512, C=3, launches=50):
    """progen_residue_head (training) and progen_residue_head_wgrad at one shape, against the HBM floor"""
    lib, st = L.load(), L.stream()
    g = torch.Generator(device='cuda').manual_seed(0)
    T = B * n
    h = torch.randn(T, d, device='cuda', generator=g).to(torch.bfloat16)
    w = torch.randn(d, C, device='cuda', generator=g) * d ** -0.5
    b = torch.zeros(C, device='cuda')
    cls = torch.randint(0, C, (T,), device='cuda', generator=g, dtype=torch.int32)
    F = lambda *s: torch.empty(*s, device='cuda')
    pred, dpred, ploss, loss, ws, dw, db = F(T * C), F(T * C), F(T), F(1), F(B * (d + 1) * C), F(d * C), F(C)
    count = torch.zeros(1, device='cuda', dtype=torch.int32)
    dy = torch.empty(T, d, device='cuda', dtype=torch.bfloat16)
    head = lambda: L.check(lib.progen_residue_head(h.data_ptr(), d, L.BF16, w.data_ptr(), b.data_ptr(), B, n, d, C,
                                                   L.TASK_CLASSIFICATION, 0, cls.data_ptr(), pred.data_ptr(),
                                                   ploss.data_ptr(), count.data_ptr(), loss.data_ptr(), dpred.data_ptr(),
                                                   dy.data_ptr(), d, st), 'residue_head')
    wgrad = lambda: L.check(lib.progen_residue_head_wgrad(h.data_ptr(), d, L.BF16, dpred.data_ptr(), 0, cls.data_ptr(), B, n,
                                                          d, C, ws.data_ptr(), dw.data_ptr(), db.data_ptr(), st), 'wgrad')
    out = {}
    for name, fn in (('head', head), ('wgrad', wgrad)):
        for _ in range(3):
            fn()
        out[name + '_us'] = timed_round(fn, launches) * 1e3
    floor_bytes = 3 * T * d * 2
    out.update(shape=dict(B=B, n=n, d=d, C=C, h_dtype='bf16'), hbm_floor_bytes=floor_bytes,
               hbm_floor_us=floor_bytes / HBM_BYTES_PER_S * 1e6)
    out['head_plus_wgrad_over_floor'] = (out['head_us'] + out['wgrad_us']) / out['hbm_floor_us']
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rank', type=int, default=16)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--skip_cfg4', action='store_true')
    args = ap.parse_args()
    L.require_device()
    res = dict(gpu=gpu_info(torch.cuda.current_device()), steps=[])
    c2 = CONFIGS['cfg2']
    for length in (384, c2['kwargs']['seq_len']):
        res['steps'].append(steps_case('cfg2', c2['kwargs'], c2['batch'], length, args.rank, args.steps, args.rounds))
    if not args.skip_cfg4:
        c4 = CONFIGS['cfg4']['kwargs']
        res['steps'].append(steps_case('cfg4', c4, 4, c4['seq_len'], args.rank, args.steps, args.rounds))
    res['kernels'] = kernels()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
