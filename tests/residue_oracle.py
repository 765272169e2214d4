"""Float64 autograd reference of per-residue fine-tuning, built on `oracle.progen_torch.forward(..., return_hidden=True)` —
test infrastructure, as the oracle is.  The head p[b, t] = h[b, t] W + b at every position of the final LayerNorm output h;
targets are indexed by position (position t >= 1 holds residue t - 1), NaN (regression) or -1 (classification) where
unlabelled.  Over the N labelled positions: regression loss sum sum_c (p - y)^2 / (C N), classification loss the mean cross
entropy.  Adapter gradients follow from the merged weight as in tests/property_oracle.py."""
import numpy as np
import torch

from oracle import progen_torch as T
from property_oracle import HEAD, merged


def residue_head_loss(h, w, b, targets, task):
    """h [B, n, d] -> (loss, predictions [B, n, C], per-position losses [B, n] (0 where unlabelled))"""
    p = h @ w + b
    if task == 'regression':
        y = torch.as_tensor(np.asarray(targets, np.float64).reshape(p.shape), dtype=p.dtype, device=p.device)
        lab = ~torch.isnan(y).all(-1)
        row = torch.where(lab, ((p - torch.nan_to_num(y)) ** 2).mean(-1), torch.zeros((), dtype=p.dtype, device=p.device))
    else:
        cls = torch.as_tensor(np.asarray(targets, np.int64), device=p.device)
        lab = cls >= 0
        row = torch.logsumexp(p, -1) - p.gather(-1, cls.clamp(min=0)[..., None])[..., 0]
        row = torch.where(lab, row, torch.zeros((), dtype=p.dtype, device=p.device))
    return row.sum() / lab.sum(), p, row


def residue_loss_and_grads(params, head, rows, targets, cfg, task, adapters=None, scale=1.0, dtype=torch.float64,
                           operand_round=None, device=None):
    """-> (float loss, adapter grads (or the base grads without adapters), head grads, predictions [B, n, C], per-position
    losses [B, n]), numpy.  With operand_round (the bf16 emulation) the head reads the rounded final LayerNorm output, as
    the engine's head reads it in the act dtype."""
    prm = T.to_torch(merged(params, adapters, scale), dtype, requires_grad=True, device=device)
    hw = torch.tensor(np.asarray(head[HEAD]['w'], np.float64), dtype=dtype, device=device, requires_grad=True)
    hb = torch.tensor(np.asarray(head[HEAD]['b'], np.float64), dtype=dtype, device=device, requires_grad=True)
    data = torch.as_tensor(np.asarray(rows).astype('int64'))
    _, h = T.forward(prm, data[:, :-1], cfg, operand_round, device, return_hidden=True)
    if operand_round is not None:
        h = operand_round(h)              # the head's input operand, like the logits GEMM's: the act dtype
    loss, p, row = residue_head_loss(h, hw, hb, targets, task)
    loss.backward()
    host = lambda t: t.detach().cpu().numpy().copy()
    grads = {m: {k: np.zeros(v.shape) if v.grad is None else host(v.grad) for k, v in d.items()} for m, d in prm.items()}
    if adapters is not None:
        grads = {m: {'lora_a': scale * grads[m]['w'] @ v['lora_b'].astype(np.float64).T,
                     'lora_b': scale * v['lora_a'].astype(np.float64).T @ grads[m]['w']} for m, v in adapters.items()}
    return float(loss.detach()), grads, {HEAD: {'w': host(hw.grad), 'b': host(hb.grad)}}, host(p), host(row)
