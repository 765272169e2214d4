"""Float64 autograd reference of property fine-tuning, built on `oracle.progen_torch.forward(..., return_hidden=True)` —
test infrastructure, as the oracle is.  The embedding is the mean of the final LayerNorm output over the loss mask
(quirk Q8: non-pad labels plus the first pad), the head p = emb W + b; regression loss sum_b sum_c (p - y)^2 / (C B),
classification loss sum_b CE_b / B.  Adapter gradients follow from the gradient wrt the merged weight W' = W + s A B as
dA = s dW' B^T, dB = s A^T dW'."""
import numpy as np
import torch

from oracle import progen_torch as T

HEAD = 'property_head'


def pooled(prm, data, cfg, operand_round=None, device=None):
    """data (B, n+1) long -> [B, d] masked mean of the final LayerNorm output (differentiable)"""
    ids, labels = data[:, :-1], data[:, 1:]
    _, h = T.forward(prm, ids, cfg, operand_round, device, return_hidden=True)
    labels = labels.to(h.device)
    mask = labels != 0
    mask = (mask | (((~mask).cumsum(-1) == 1) & ~mask)).to(h.dtype)
    return (h * mask[..., None]).sum(1) / mask.sum(1, keepdim=True)


def head_loss(emb, w, b, targets, task, global_batch=None):
    """-> (loss, predictions [B, C], per-row losses [B])"""
    p = emb @ w + b
    if task == 'regression':
        y = torch.as_tensor(np.asarray(targets, np.float64).reshape(p.shape), dtype=p.dtype, device=p.device)
        row = ((p - y) ** 2).mean(-1)
    else:
        cls = torch.as_tensor(np.asarray(targets, np.int64), device=p.device)
        row = torch.logsumexp(p, -1) - p.gather(-1, cls[:, None])[:, 0]
    return row.sum() / (global_batch or p.shape[0]), p, row


def merged(params, adapters, scale):
    out = {m: dict(v) for m, v in params.items()}
    for m, v in (adapters or {}).items():
        out[m]['w'] = params[m]['w'].astype(np.float64) + scale * (v['lora_a'].astype(np.float64) @ v['lora_b'].astype(np.float64))
    return out


def property_loss_and_grads(params, head, rows, targets, cfg, task, adapters=None, scale=1.0, dtype=torch.float64,
                            operand_round=None, device=None):
    """-> (float loss, adapter grads (or the base grads without adapters), head grads, predictions [B, C], row losses [B],
    embedding [B, d]), numpy"""
    prm = T.to_torch(merged(params, adapters, scale), dtype, requires_grad=True, device=device)
    hw = torch.tensor(np.asarray(head[HEAD]['w'], np.float64), dtype=dtype, device=device, requires_grad=True)
    hb = torch.tensor(np.asarray(head[HEAD]['b'], np.float64), dtype=dtype, device=device, requires_grad=True)
    data = torch.as_tensor(np.asarray(rows).astype('int64'))
    emb = pooled(prm, data, cfg, operand_round, device)
    loss, p, row = head_loss(emb, hw, hb, targets, task)
    loss.backward()
    host = lambda t: t.detach().cpu().numpy().copy()
    # the logits head does not reach the loss: its gradient is zero
    grads = {m: {k: np.zeros(v.shape) if v.grad is None else host(v.grad) for k, v in d.items()} for m, d in prm.items()}
    if adapters is not None:
        grads = {m: {'lora_a': scale * grads[m]['w'] @ v['lora_b'].astype(np.float64).T,
                     'lora_b': scale * v['lora_a'].astype(np.float64).T @ grads[m]['w']} for m, v in adapters.items()}
    return float(loss.detach()), grads, {HEAD: {'w': host(hw.grad), 'b': host(hb.grad)}}, host(p), host(row), host(emb)
