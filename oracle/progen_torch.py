"""Torch-CPU autograd twin of `oracle/progen_ref.py` — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Same algorithm (reference lines cited in progen_ref.py), batched over sequences and differentiable, so that
gradient goldens exist (the reference obtains them from `jax.value_and_grad`, utils.py:72).  It is validated
against the NumPy oracle (forward) and finite differences (backward) in tests/test_oracle_golden.py.
It is also the timed CPU baseline of bench.py (`cpu_baseline.kind == "port"`, all host cores through torch's
intra-op threads), because the reference's Jax path cannot be installed here or on the GPU box.

`operand_round` (optional) is applied to every GEMM / attention operand; passing a bf16 round-trip predicts the
error of a bf16-operand / fp32-accumulate engine on CPU before spending GPU time.

`device` (optional, default CPU) runs the same algorithm on another torch device, for shapes where float64 on the host is
too slow (tests/test_gpu_large_configs.py).  Tables (rotary) are computed on the host in float64 either way and then moved,
so only the GEMM / reduction order of the device differs.
"""
import math
import torch

from .progen_ref import P, layer_kinds, ATTN_MASK_VALUE, LN_EPS


def to_torch(params, dtype=torch.float64, requires_grad=False, device=None):
    out = {}
    for m, d in params.items():
        out[m] = {}
        for k, v in d.items():
            t = torch.tensor(v, dtype=dtype, device=device)
            t.requires_grad_(requires_grad)
            out[m][k] = t
    return out


def _ln(x, scale):
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + LN_EPS) * scale


def _shift(x):
    half = (x.shape[-1] + 1) // 2
    xs = torch.nn.functional.pad(x[:, :-1, :half], (0, 0, 1, 0))
    return torch.cat((xs, x[..., half:]), dim=-1)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def _rotary_tables(n, dh, dtype):
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dh, 2, dtype=torch.float64) / dh))
    ang = torch.arange(n, dtype=torch.float64)[:, None] * inv_freq[None, :]
    ang = ang.repeat_interleave(2, dim=-1)
    return torch.sin(ang).to(dtype), torch.cos(ang).to(dtype)


def _rot(x, sin, cos):
    x2 = torch.stack((-x[..., 1::2], x[..., 0::2]), dim=-1).flatten(-2)
    return x * cos + x2 * sin


def forward(prm, ids, cfg, operand_round=None, device=None, return_hidden=False, probe=None):
    """prm: nested dict of tensors on `device` (default CPU); ids: (B, n) long -> logits (B, n, V), or with
    `return_hidden` (logits, the final LayerNorm output (B, n, d): the head's input, which scoring pools).
    `probe` (optional dict) receives, per layer, lists of intermediate tensors without changing any result: 'resid' the
    residual stream entering the layer (and, last, the stream entering the final LayerNorm), 'attn' the attention
    probabilities (B, h, W, w, 2w), 'gelu_in' the GELU input (the gate half for GLU layers)."""
    r = operand_round or (lambda t: t)
    dev = torch.device('cpu') if device is None else torch.device(device)
    ids = ids.to(dev)
    B, n = ids.shape
    h, dh, w = cfg['heads'], cfg['dim_head'], cfg['window_size']
    W = n // w
    x = prm[P + 'embed']['embeddings'][ids.clamp(0, cfg['num_tokens'] - 1)]     # jax gather clamps
    dtype = x.dtype
    sin, cos = (t.to(dev) for t in _rotary_tables(n, dh, dtype))
    mask = torch.tril(torch.ones(w, 2 * w, dtype=torch.bool, device=dev), w)
    keep = (lambda key, t: probe.setdefault(key, []).append(t.detach())) if probe is not None else (lambda key, t: None)
    for i, kind in enumerate(layer_kinds(cfg)):
        a = P + f'attn{i}/~/'
        keep('resid', x)
        y = _ln(x, prm[a + 'layer_norm']['scale'])
        if cfg['shift_tokens']:
            y = _shift(y)
        qkv = r(y) @ r(prm[a + 'linear']['w'])
        q, k, v = qkv.chunk(3, dim=-1)
        q, k, v = (t.reshape(B, n, h, dh).transpose(1, 2) for t in (q, k, v))
        q, k, v = (r(_rot(t, sin, cos)) for t in (q, k, v))
        q, k, v = (t.reshape(B, h, W, w, dh) for t in (q, k, v))
        k, v = (torch.cat((torch.zeros_like(t[:, :, :1]), t), dim=2) for t in (k, v))
        k, v = (torch.cat((t[:, :, :-1], t[:, :, 1:]), dim=3) for t in (k, v))
        sim = torch.einsum('bhwid,bhwjd->bhwij', q, k) * (dh ** -0.5)
        sim = torch.where(mask, sim, torch.full_like(sim, ATTN_MASK_VALUE))
        attn = torch.softmax(sim, dim=-1)
        keep('attn', attn)
        o = torch.einsum('bhwij,bhwjd->bhwid', r(attn), v)
        o = o.reshape(B, h, n, dh).transpose(1, 2).reshape(B, n, h * dh)
        x = x + r(o) @ r(prm[a + 'linear_1']['w']) + prm[a + 'linear_1']['b']

        f = P + f'ff{i}/~/'
        y = _ln(x, prm[f + 'layer_norm']['scale'])
        if cfg['shift_tokens']:
            y = _shift(y)
        u = r(y) @ r(prm[f + 'linear']['w']) + prm[f + 'linear']['b']
        if kind == 'glu':
            val, gate = u.chunk(2, dim=-1)
            keep('gelu_in', gate)
            u = val * _gelu(gate)
        else:
            keep('gelu_in', u)
            u = _gelu(u)
        if kind == 'sgu':
            xs, gate = u.chunk(2, dim=-1)
            gate = _ln(gate, prm[f + 'sgu/~/layer_norm']['scale'])
            wts = prm[f + 'sgu']['spatial_weights'] * torch.tril(torch.ones(n, n, dtype=dtype, device=dev))
            gate = torch.einsum('mk,bkd->bmd', r(wts), r(gate)) + prm[f + 'sgu']['spatial_biases']
            u = xs * gate
            u = r(u) @ r(prm[f + 'sgu/~/linear']['w']) + prm[f + 'sgu/~/linear']['b']
        x = x + r(u) @ r(prm[f + 'linear_1']['w']) + prm[f + 'linear_1']['b']
    keep('resid', x)
    x = _ln(x, prm[P + 'layer_norm']['scale'])
    logits = r(x) @ r(prm[P + 'linear']['w']) + prm[P + 'linear']['b']
    return (logits, x) if return_hidden else logits


def cross_entropy(logits, targets, ignore_index=0):
    logp = torch.log_softmax(logits, dim=-1)
    nll = logp.gather(-1, targets[..., None])[..., 0]
    mask = targets != ignore_index
    eos = ((~mask).cumsum(-1) == 1) & ~mask
    mask = (mask | eos).to(logits.dtype)
    return -(nll * mask).sum(-1) / mask.sum(-1)


def batch_loss(prm, data, cfg, operand_round=None, device=None):
    """data: (B, n+1) long -> scalar (mean over rows of per-row CE), utils.py:61-76."""
    ids, labels = data[:, :-1], data[:, 1:]
    logits = forward(prm, ids, cfg, operand_round, device)
    return cross_entropy(logits, labels.to(logits.device)).mean()


def loss_and_grads(params_np, data_np, cfg, dtype=torch.float64, operand_round=None, device=None):
    """`operand_round=bf16_round` (with dtype=float32) is the CPU emulation of a bf16-operand / fp32-accumulate engine:
    autograd sends the gradients through the same casts, so the backward GEMM operands are rounded as well.
    `device` (default CPU) is where the evaluation runs; the gradients come back as host numpy arrays."""
    prm = to_torch(params_np, dtype, requires_grad=True, device=device)
    data = torch.as_tensor(data_np.astype('int64'))
    loss = batch_loss(prm, data, cfg, operand_round, device)
    loss.backward()
    grads = {m: {k: v.grad.cpu().numpy().copy() for k, v in d.items()} for m, d in prm.items()}
    return float(loss.detach()), grads


def bf16_round(t):
    return t.to(torch.bfloat16).to(t.dtype)
