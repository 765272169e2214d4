"""Float64 autograd reference of the preference (DPO) loss, built on `oracle.progen_torch.forward` — test infrastructure,
as the oracle is.  Rows and masks follow `ProGen.preference_loss_and_grad`: pair i is (chosen[i], rejected[i]), s(x) the
sum of the label log-probabilities under the loss mask (quirk Q8: non-pad labels plus the first pad)."""
import numpy as np
import torch

from oracle import progen_torch as T


def seq_log_likelihood(prm, data, cfg, operand_round=None, device=None):
    """data (B, n+1) long -> [B] sum over counted positions of log_softmax(logits)[label] (differentiable)"""
    ids, labels = data[:, :-1], data[:, 1:]
    logits = T.forward(prm, ids, cfg, operand_round, device)
    labels = labels.to(logits.device)
    logp = torch.log_softmax(logits, dim=-1).gather(-1, labels[..., None])[..., 0]
    mask = labels != 0
    mask = mask | (((~mask).cumsum(-1) == 1) & ~mask)
    return (logp * mask.to(logp.dtype)).sum(-1)


def preference_loss(prm, chosen, rejected, ref_chosen, ref_rejected, cfg, beta, global_pairs=None, operand_round=None,
                    device=None):
    """-> (loss = sum_i softplus(-z_i) / global_pairs (default P), (s_c, s_r, z, per-pair loss))"""
    P = chosen.shape[0]
    s = seq_log_likelihood(prm, torch.cat([chosen, rejected]), cfg, operand_round, device)
    s_c, s_r = s[:P], s[P:]
    rc = torch.as_tensor(np.asarray(ref_chosen, np.float64), dtype=s.dtype, device=s.device)
    rr = torch.as_tensor(np.asarray(ref_rejected, np.float64), dtype=s.dtype, device=s.device)
    z = beta * ((s_c - rc) - (s_r - rr))
    pair = torch.nn.functional.softplus(-z)
    return pair.sum() / (global_pairs or P), (s_c, s_r, z, pair)


def preference_loss_and_grads(params_np, chosen_np, rejected_np, ref_chosen, ref_rejected, cfg, beta, dtype=torch.float64,
                              global_pairs=None, operand_round=None, device=None):
    """-> (float loss, haiku-shaped numpy gradients, stats dict of numpy [P]: policy_chosen, policy_rejected, margin, loss)"""
    prm = T.to_torch(params_np, dtype, requires_grad=True, device=device)
    c = torch.as_tensor(np.asarray(chosen_np).astype('int64'))
    r = torch.as_tensor(np.asarray(rejected_np).astype('int64'))
    loss, (s_c, s_r, z, pair) = preference_loss(prm, c, r, ref_chosen, ref_rejected, cfg, beta, global_pairs,
                                                operand_round, device)
    loss.backward()
    grads = {m: {k: v.grad.cpu().numpy().copy() for k, v in d.items()} for m, d in prm.items()}
    host = lambda t: t.detach().cpu().numpy().copy()
    stats = dict(policy_chosen=host(s_c), policy_rejected=host(s_r), margin=host(z), loss=host(pair))
    return float(loss.detach()), grads, stats
