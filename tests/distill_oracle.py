"""Float64 reference of distillation (DESIGN.md §3.13) — test infrastructure, as the oracle is.

`distill_head` is the head alone in NumPy: student logits s [B, n, V], teacher logits z [B, n, V], labels [B, n]; per
counted position (the loss mask of `cross_entropy`, Q8) KL_t = KL(softmax(z / tau) || softmax(s / tau)) and CE_t =
-log_softmax(s)[label_t]; per row their means over the counted positions; loss = inv_batch sum_b [(1 - alpha) tau^2 KL_b +
alpha CE_b], and its gradient with respect to s.  `distill_loss_and_grads` is the model-level twin on
`oracle.progen_torch.forward`, student and teacher each at its own config."""
import numpy as np
import torch

from oracle import progen_torch as T


def loss_mask(labels):
    """labels [B, n] -> float64 mask [B, n]: non-pad labels plus the first pad (quirk Q8)"""
    labels = np.asarray(labels)
    pad = labels == 0
    eos = (np.cumsum(pad, axis=-1) == 1) & pad
    return (~pad | eos).astype(np.float64)


def _log_softmax(x):
    m = x.max(-1, keepdims=True)
    return x - m - np.log(np.exp(x - m).sum(-1, keepdims=True))


def distill_head(s, z, labels, tau, alpha, inv_batch=None):
    """-> (loss, dlogits [B, n, V], stats [B, 2] = (KL_b, CE_b)), all float64; inv_batch default 1 / B"""
    s, z = np.asarray(s, np.float64), np.asarray(z, np.float64)
    labels = np.asarray(labels)
    B, n, V = s.shape
    inv_batch = 1.0 / B if inv_batch is None else inv_batch
    m = loss_mask(labels)
    c = m.sum(-1)
    lq, lp = _log_softmax(s / tau), _log_softmax(z / tau)
    p = np.exp(lp)
    kl = np.where(p > 0, p * (lp - lq), 0.0).sum(-1)
    ls = _log_softmax(s)
    lab = np.clip(labels, 0, V - 1)
    ce = -np.take_along_axis(ls, lab[..., None], -1)[..., 0]
    stats = np.stack([(m * kl).sum(-1) / c, (m * ce).sum(-1) / c], -1)
    loss = inv_batch * ((1 - alpha) * tau ** 2 * stats[:, 0] + alpha * stats[:, 1]).sum()
    onehot = np.eye(V)[lab]
    w = (inv_batch * m / c[:, None])[..., None]
    grad = w * ((1 - alpha) * tau * (np.exp(lq) - p) + alpha * (np.exp(ls) - onehot))
    return float(loss), grad, stats


def distill_loss_and_grads(params, cfg, teacher_params, teacher_cfg, rows, tau, alpha, adapters=None, scale=1.0,
                           dtype=torch.float64, operand_round=None):
    """-> (float loss, grads (the adapters' with adapters), stats [B, 2]) of the student on rows (B, n+1); the teacher
    runs on the same ids, zero-padded to its seq_len"""
    from property_oracle import merged
    rows = np.asarray(rows).astype(np.int64)
    B, n = rows.shape[0], cfg['seq_len']
    ids = torch.as_tensor(rows[:, :-1])
    tid = torch.zeros((B, teacher_cfg['seq_len']), dtype=torch.int64)
    tid[:, :n] = ids
    with torch.no_grad():
        z = T.forward(T.to_torch(teacher_params, dtype), tid, teacher_cfg, operand_round)[:, :n]
    prm = T.to_torch(merged(params, adapters, scale), dtype, requires_grad=True)
    s = T.forward(prm, ids, cfg, operand_round)
    labels = torch.as_tensor(rows[:, 1:])
    lq, lp = torch.log_softmax(s / tau, -1), torch.log_softmax(z / tau, -1)
    p = lp.exp()
    kl = torch.where(p > 0, p * (lp - lq), torch.zeros((), dtype=s.dtype)).sum(-1)
    m = torch.as_tensor(loss_mask(rows[:, 1:]), dtype=s.dtype)
    ce_t = -torch.log_softmax(s, -1).gather(-1, labels.clamp(0, s.shape[-1] - 1)[..., None])[..., 0]
    klb, ceb = (m * kl).sum(-1) / m.sum(-1), (m * ce_t).sum(-1) / m.sum(-1)
    loss = ((1 - alpha) * tau ** 2 * klb + alpha * ceb).mean()
    loss.backward()
    host = lambda t: t.detach().cpu().numpy().copy()
    grads = {mm: {k: np.zeros(v.shape) if v.grad is None else host(v.grad) for k, v in d.items()} for mm, d in prm.items()}
    if adapters is not None:
        grads = {mm: {'lora_a': scale * grads[mm]['w'] @ v['lora_b'].astype(np.float64).T,
                      'lora_b': scale * v['lora_a'].astype(np.float64).T @ grads[mm]['w']} for mm, v in adapters.items()}
    return float(loss.detach()), grads, np.stack([host(klb), host(ceb)], -1)
