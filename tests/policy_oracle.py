"""Float64 reference of the policy-gradient objective (DESIGN.md §3.14) — test infrastructure, as the oracle is.

`policy_head` is the head alone in NumPy: policy logits s [B, n, V], reference logits z [B, n, V] (or None with beta =
0), labels [B, n], spans [B, 2] and advantages [B]; per position t of row b's span, logp_t = log_softmax(s_t)[label_t]
and KL_t = KL(softmax(s_t) || softmax(z_t)) (0 with beta = 0, where the reference is not read); L_b = mean over the
span of (-A_b logp_t + beta KL_t); loss = inv_rows sum_b L_b, and its gradient with respect to s.  `policy_loss_and_grads` is the model-level twin on
`oracle.progen_torch.forward`, autograd through the same loss."""
import numpy as np
import torch

from oracle import progen_torch as T


def _log_softmax(x):
    m = x.max(-1, keepdims=True)
    return x - m - np.log(np.exp(x - m).sum(-1, keepdims=True))


def span_mask(span, B, n):
    """span [B, 2] -> float64 mask [B, n] of lo_b <= t < hi_b"""
    t = np.arange(n)[None, :]
    span = np.asarray(span)
    return ((t >= span[:, :1]) & (t < span[:, 1:])).astype(np.float64)


def policy_head(s, z, labels, span, adv, beta, inv_rows=None):
    """-> (loss, dlogits [B, n, V], stats [B, 3] = (mean logp, mean KL, N_b)), all float64; inv_rows default 1 / B"""
    s = np.asarray(s, np.float64)
    B, n, V = s.shape
    inv_rows = 1.0 / B if inv_rows is None else inv_rows
    m = span_mask(span, B, n)
    N = m.sum(-1)
    lpi = _log_softmax(s)
    pi = np.exp(lpi)
    lab = np.clip(np.asarray(labels), 0, V - 1)
    logp = np.take_along_axis(lpi, lab[..., None], -1)[..., 0]
    if z is None or beta == 0:                              # with beta = 0 the reference is not read: KL_t = 0
        d = np.zeros_like(lpi)
    else:
        d = lpi - _log_softmax(np.asarray(z, np.float64))
    kl = np.where(pi > 0, pi * d, 0.0).sum(-1)
    adv = np.asarray(adv, np.float64)
    stats = np.stack([(m * logp).sum(-1) / N, (m * kl).sum(-1) / N, N], -1)
    loss = inv_rows * (-adv * stats[:, 0] + beta * stats[:, 1]).sum()
    w = (inv_rows * m / N[:, None])[..., None]
    onehot = np.eye(V)[lab]
    grad = w * (adv[:, None, None] * (pi - onehot) + beta * pi * (d - kl[..., None]))
    return float(loss), grad, stats


def policy_loss_and_grads(params, cfg, ref_params, ref_cfg, rows, span, adv, beta, adapters=None, scale=1.0,
                          dtype=torch.float64, operand_round=None):
    """-> (float loss, grads (the adapters' with adapters), stats [B, 3]) of the policy on rows (B, n+1); the reference
    (None with beta = 0) runs on the same ids, zero-padded to its seq_len"""
    from property_oracle import merged
    rows = np.asarray(rows).astype(np.int64)
    B, n = rows.shape[0], cfg['seq_len']
    ids = torch.as_tensor(rows[:, :-1])
    prm = T.to_torch(merged(params, adapters, scale), dtype, requires_grad=True)
    s = T.forward(prm, ids, cfg, operand_round)
    lpi = torch.log_softmax(s, -1)
    labels = torch.as_tensor(rows[:, 1:]).clamp(0, s.shape[-1] - 1)
    logp = lpi.gather(-1, labels[..., None])[..., 0]
    if beta > 0:
        tid = torch.zeros((B, ref_cfg['seq_len']), dtype=torch.int64)
        tid[:, :n] = ids
        with torch.no_grad():
            z = T.forward(T.to_torch(ref_params, dtype), tid, ref_cfg, operand_round)[:, :n]
        pi = lpi.exp()
        kl = torch.where(pi > 0, pi * (lpi - torch.log_softmax(z, -1)), torch.zeros((), dtype=s.dtype)).sum(-1)
    else:
        kl = torch.zeros_like(logp)
    m = torch.as_tensor(span_mask(span, B, n), dtype=s.dtype)
    N = m.sum(-1)
    a = torch.as_tensor(np.asarray(adv, np.float64), dtype=s.dtype)
    lpb, klb = (m * logp).sum(-1) / N, (m * kl).sum(-1) / N
    loss = (-a * lpb + beta * klb).mean()
    loss.backward()
    host = lambda t: t.detach().cpu().numpy().copy()
    grads = {mm: {k: np.zeros(v.shape) if v.grad is None else host(v.grad) for k, v in d.items()} for mm, d in prm.items()}
    if adapters is not None:
        grads = {mm: {'lora_a': scale * grads[mm]['w'] @ v['lora_b'].astype(np.float64).T,
                      'lora_b': scale * v['lora_a'].astype(np.float64).T @ grads[mm]['w']} for mm, v in adapters.items()}
    return float(loss.detach()), grads, np.stack([host(lpb), host(klb), host(N)], -1)
