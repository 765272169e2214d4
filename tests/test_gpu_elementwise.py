"""HBM kernels + fp32 attention + optimizer through the C ABI, each against a plain torch float64 reference of the same
op (and the NumPy oracle for the optimizer chain)."""
import math
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _L():
    from progen_b200 import lib as L
    L.require_device()
    return L


def ln_ref(x, scale):
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + 1e-5) * scale


def shift_ref(y, n):
    B = y.shape[0] // n
    y3 = y.view(B, n, -1)
    half = y3.shape[-1] // 2
    ys = torch.nn.functional.pad(y3[:, :-1, :half], (0, 0, 1, 0))
    return torch.cat((ys, y3[..., half:]), dim=-1).reshape(y.shape)


@pytest.mark.parametrize('act', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('shift', [0, 1])
@pytest.mark.parametrize('d', [64, 512, 1536])
def test_ln_shift_fwd_bwd(act, shift, d):
    L = _L()
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(d + shift)
    B, n = 3, 24
    T = B * n
    x = torch.randn(T, d, generator=g, device=dev) * 2 + 0.5
    scale = torch.randn(d, generator=g, device=dev)
    y = torch.empty(T, d, device=dev, dtype=act)
    mean = torch.empty(T, device=dev)
    rstd = torch.empty(T, device=dev)
    L.check(L.load().progen_ln_shift_fwd(x.data_ptr(), d, L.F32, scale.data_ptr(), y.data_ptr(), d, L.dt(y), mean.data_ptr(),
                                         rstd.data_ptr(), T, d, n, shift, L.stream()))
    xd = x.double().requires_grad_(True)
    sd = scale.double().requires_grad_(True)
    ref = ln_ref(xd, sd)
    if shift:
        ref = shift_ref(ref, n)
    tol = 1e-5 if act == torch.float32 else 2e-2
    assert (y.double() - ref).abs().max().item() < tol * max(1.0, ref.abs().max().item())
    # backward (residual mode): dres += dx
    dy = torch.randn(T, d, generator=g, device=dev).to(act)
    dres0 = torch.randn(T, d, generator=g, device=dev)
    dres = dres0.clone()
    dres_lp = torch.empty(T, d, device=dev, dtype=act)
    dscale = torch.zeros(d, device=dev)
    csum = torch.zeros(d, device=dev)
    L.check(L.load().progen_ln_shift_bwd(dy.data_ptr(), d, L.dt(dy), x.data_ptr(), d, L.F32, scale.data_ptr(), mean.data_ptr(),
                                         rstd.data_ptr(), dres.data_ptr(), dres_lp.data_ptr(), d, dscale.data_ptr(), csum.data_ptr(),
                                         T, d, n, shift, 1, L.stream()))
    ref.backward(dy.double())
    assert (dres.double() - (dres0.double() + xd.grad)).abs().max().item() < 1e-4 * max(1.0, xd.grad.abs().max().item())
    assert (dscale.double() - sd.grad).abs().max().item() < 1e-3 * max(1.0, sd.grad.abs().max().item())
    assert (dres_lp.double() - dres.double()).abs().max().item() <= (1e-6 if act == torch.float32 else 0.05)
    assert (csum.double() - dres.double().sum(0)).abs().max().item() < 1e-3 * max(1.0, dres.double().sum(0).abs().max().item())


def test_ln_strided_act_input():
    """SGU LayerNorm: act-dtype input taken from the second half of a wider buffer, non-residual backward."""
    L = _L()
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(0)
    T, C = 40, 256
    a = torch.randn(T, 2 * C, generator=g, device=dev).bfloat16()
    scale = torch.randn(C, generator=g, device=dev)
    y = torch.empty(T, C, device=dev, dtype=torch.bfloat16)
    mean = torch.empty(T, device=dev)
    rstd = torch.empty(T, device=dev)
    gate = a[:, C:]
    L.check(L.load().progen_ln_shift_fwd(gate.data_ptr(), 2 * C, L.BF16, scale.data_ptr(), y.data_ptr(), C, L.BF16,
                                         mean.data_ptr(), rstd.data_ptr(), T, C, T, 0, L.stream()))
    xd = gate.double().requires_grad_(True)
    sd = scale.double().requires_grad_(True)
    ref = ln_ref(xd, sd)
    assert (y.double() - ref).abs().max().item() < 2e-2 * ref.abs().max().item()
    dy = torch.randn(T, C, generator=g, device=dev).bfloat16()
    da = torch.zeros(T, 2 * C, device=dev, dtype=torch.bfloat16)
    dscale = torch.zeros(C, device=dev)
    L.check(L.load().progen_ln_shift_bwd(dy.data_ptr(), C, L.BF16, gate.data_ptr(), 2 * C, L.BF16, scale.data_ptr(),
                                         mean.data_ptr(), rstd.data_ptr(), 0, da[:, C:].data_ptr(), 2 * C, dscale.data_ptr(), 0,
                                         T, C, T, 0, 0, L.stream()))
    ref.backward(dy.double())
    assert (da[:, C:].double() - xd.grad).abs().max().item() < 2e-2 * xd.grad.abs().max().item()
    assert da[:, :C].abs().max().item() == 0
    assert (dscale.double() - sd.grad).abs().max().item() < 1e-3 * sd.grad.abs().max().item()


@pytest.mark.parametrize('act', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('d,B,n', [(512, 8, 1024), (1024, 5, 768), (128, 16, 64), (1536, 4, 768), (2048, 3, 516)])
def test_ln_bwd_stream_path_residual(act, d, B, n):
    """Shapes the bulk-copy streaming kernel (ln_stream.cu) takes: many chunks per CTA so every stage wraps several
    times, sequence boundaries inside chunks' look-ahead rows, residual accumulate + low-precision copy + column sums."""
    L = _L()
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(d + n)
    T = B * n
    x = torch.randn(T, d, generator=g, device=dev) * 1.5 - 0.3
    scale = torch.randn(d, generator=g, device=dev)
    y = torch.empty(T, d, device=dev, dtype=act)
    mean = torch.empty(T, device=dev)
    rstd = torch.empty(T, device=dev)
    L.check(L.load().progen_ln_shift_fwd(x.data_ptr(), d, L.F32, scale.data_ptr(), y.data_ptr(), d, L.dt(y), mean.data_ptr(),
                                         rstd.data_ptr(), T, d, n, 1, L.stream()))
    xd = x.double().requires_grad_(True)
    sd = scale.double().requires_grad_(True)
    ref = shift_ref(ln_ref(xd, sd), n)
    dy = torch.randn(T, d, generator=g, device=dev).to(act)
    dres0 = torch.randn(T, d, generator=g, device=dev)
    dres = dres0.clone()
    dres_lp = torch.full((T, d), float('nan'), device=dev, dtype=act)
    dscale = torch.zeros(d, device=dev)
    csum = torch.zeros(d, device=dev)
    for use_lp in (True, False):
        dres.copy_(dres0); dscale.zero_(); csum.zero_()
        L.check(L.load().progen_ln_shift_bwd(dy.data_ptr(), d, L.dt(dy), x.data_ptr(), d, L.F32, scale.data_ptr(), mean.data_ptr(),
                                             rstd.data_ptr(), dres.data_ptr(), dres_lp.data_ptr() if use_lp else 0, d,
                                             dscale.data_ptr(), csum.data_ptr(), T, d, n, 1, 1, L.stream()))
        if xd.grad is None:
            ref.backward(dy.double())
        gs = max(1.0, xd.grad.abs().max().item())
        assert (dres.double() - (dres0.double() + xd.grad)).abs().max().item() < 1e-4 * gs
        assert (dscale.double() - sd.grad).abs().max().item() < 1e-3 * max(1.0, sd.grad.abs().max().item())
        assert (dres_lp.double() - dres.double()).abs().max().item() <= (1e-6 if act == torch.float32 else 0.06)
        cs_ref = dres.double().sum(0)
        assert (csum.double() - cs_ref).abs().max().item() < 1e-3 * max(1.0, cs_ref.abs().max().item())


def test_ln_bwd_stream_path_strided_nonresidual():
    """SGU LayerNorm backward at a streaming-kernel shape: bf16 input/output taken as column slices of wider buffers."""
    L = _L()
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(3)
    T, C = 8 * 1024, 1024
    a = torch.randn(T, 2 * C, generator=g, device=dev).bfloat16()
    scale = torch.randn(C, generator=g, device=dev)
    y = torch.empty(T, C, device=dev, dtype=torch.bfloat16)
    mean = torch.empty(T, device=dev)
    rstd = torch.empty(T, device=dev)
    gate = a[:, C:]
    L.check(L.load().progen_ln_shift_fwd(gate.data_ptr(), 2 * C, L.BF16, scale.data_ptr(), y.data_ptr(), C, L.BF16,
                                         mean.data_ptr(), rstd.data_ptr(), T, C, 1024, 0, L.stream()))
    xd = gate.double().requires_grad_(True)
    sd = scale.double().requires_grad_(True)
    ref = ln_ref(xd, sd)
    dy = torch.randn(T, C, generator=g, device=dev).bfloat16()
    da = torch.zeros(T, 2 * C, device=dev, dtype=torch.bfloat16)
    dscale = torch.zeros(C, device=dev)
    L.check(L.load().progen_ln_shift_bwd(dy.data_ptr(), C, L.BF16, gate.data_ptr(), 2 * C, L.BF16, scale.data_ptr(),
                                         mean.data_ptr(), rstd.data_ptr(), 0, da[:, C:].data_ptr(), 2 * C, dscale.data_ptr(), 0,
                                         T, C, 1024, 0, 0, L.stream()))
    ref.backward(dy.double())
    assert (da[:, C:].double() - xd.grad).abs().max().item() < 2e-2 * xd.grad.abs().max().item()
    assert da[:, :C].abs().max().item() == 0
    assert (dscale.double() - sd.grad).abs().max().item() < 2e-3 * sd.grad.abs().max().item()


def test_embed_fwd_bwd_and_colsum():
    L = _L()
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(0)
    T, d, V = 5000, 96, 256
    tok = torch.randint(0, V, (T,), generator=g, device=dev, dtype=torch.int32)
    table = torch.randn(V, d, generator=g, device=dev)
    x = torch.empty(T, d, device=dev)
    L.check(L.load().progen_embed_fwd(tok.data_ptr(), table.data_ptr(), x.data_ptr(), T, d, V, L.stream()))
    assert torch.equal(x, table[tok.long()])
    dx = torch.randn(T, d, generator=g, device=dev)
    dtab = torch.zeros(V, d, device=dev)
    L.check(L.load().progen_embed_bwd(tok.data_ptr(), dx.data_ptr(), dtab.data_ptr(), T, d, V, L.stream()))
    ref = torch.zeros(V, d, device=dev, dtype=torch.float64).index_add_(0, tok.long(), dx.double())
    assert (dtab.double() - ref).abs().max().item() < 1e-4
    for dtype in (torch.float32, torch.bfloat16):
        m = dx.to(dtype)
        out = torch.zeros(d, device=dev)
        L.check(L.load().progen_colsum(m.data_ptr(), d, L.dt(m), out.data_ptr(), T, d, L.stream()))
        assert (out.double() - m.double().sum(0)).abs().max().item() < 1e-3


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_cross_entropy_fwd_bwd(dtype):
    L = _L()
    from oracle import progen_ref as O
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(0)
    B, n, V = 4, 96, 256
    logits = (torch.randn(B * n, V, generator=g, device=dev) * 3).to(dtype)
    labels = torch.randint(0, V, (B, n), generator=g, device=dev, dtype=torch.int32)
    labels[1, 40:] = 0                      # EOS then padding
    labels[2, 0] = 0                        # first label is already the pad/EOS token
    labels[3] = 0                           # everything pad: only the first position counts
    w = torch.empty(B * n, device=dev)
    loss = torch.zeros(1, device=dev)
    dlogits = torch.empty_like(logits)
    L.check(L.load().progen_ce_fwd_bwd(logits.data_ptr(), L.dt(logits), labels.data_ptr(), w.data_ptr(), loss.data_ptr(),
                                       dlogits.data_ptr(), L.dt(dlogits), B, n, V, 1.0 / B, L.stream()))
    lg = logits.double().view(B, n, V).requires_grad_(True)
    ref = sum(float(O.cross_entropy(lg[b].detach().cpu().numpy(), labels[b].cpu().numpy())) for b in range(B)) / B
    assert abs(loss.item() - ref) < 1e-4 * max(1.0, abs(ref))
    # gradient reference through torch
    logp = torch.log_softmax(lg, -1)
    nll = -logp.gather(-1, labels.long()[..., None])[..., 0]
    mask = torch.as_tensor(np.stack([O.loss_mask(labels[b].cpu().numpy()) for b in range(B)]), device=dev).double()
    ((nll * mask).sum(-1) / mask.sum(-1)).mean().backward()
    tol = 1e-6 if dtype == torch.float32 else 2e-3 * lg.grad.abs().max().item() + 1e-5
    assert (dlogits.double().view(B, n, V) - lg.grad).abs().max().item() < tol


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_rotary_bwd_sgu_gate_gelu(dtype):
    L = _L()
    from gemm_cases import rotary_tables, gelu_grad
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(0)
    B, n, h, dh = 2, 48, 3, 32
    T, N = B * n, 3 * h * dh
    sin, cos = rotary_tables(n, dh, dev)
    x = torch.randn(T, N, generator=g, device=dev).to(dtype)
    xd = x.double().requires_grad_(True)
    pos = torch.arange(T, device=dev) % n
    s = sin.double()[pos].repeat_interleave(2, dim=-1).repeat(1, N // dh)
    c = cos.double()[pos].repeat_interleave(2, dim=-1).repeat(1, N // dh)
    rot = torch.stack((-xd[:, 1::2], xd[:, 0::2]), dim=-1).flatten(-2)
    y = xd * c + rot * s
    dy = torch.randn(T, N, generator=g, device=dev).to(dtype)
    y.backward(dy.double())
    buf = dy.clone()
    L.check(L.load().progen_rotary_bwd(buf.data_ptr(), N, L.dt(buf), sin.data_ptr(), cos.data_ptr(), T, N, n, dh, L.stream()))
    tol = 1e-5 if dtype == torch.float32 else 3e-2
    assert (buf.double() - xd.grad).abs().max().item() < tol
    # SGU gate fwd / bwd
    C = 64
    a = torch.randn(T, 2 * C, generator=g, device=dev).to(dtype)       # xs = a[:, :C]
    gp = torch.randn(T, C, generator=g, device=dev).to(dtype)
    bias = torch.randn(n, generator=g, device=dev)
    out = torch.empty(T, C, device=dev, dtype=dtype)
    L.check(L.load().progen_sgu_gate_fwd(a.data_ptr(), 2 * C, gp.data_ptr(), C, bias.data_ptr(), out.data_ptr(), C, L.dt(a), T, C,
                                         n, L.stream()))
    xs = a[:, :C].double().requires_grad_(True)
    gpd = gp.double().requires_grad_(True)
    bd = bias.double().requires_grad_(True)
    ref = xs * (gpd + bd[pos][:, None])
    assert (out.double() - ref).abs().max().item() < (1e-5 if dtype == torch.float32 else 5e-2)
    ds = torch.randn(T, C, generator=g, device=dev).to(dtype)
    ref.backward(ds.double())
    da = torch.zeros(T, 2 * C, device=dev, dtype=dtype)
    dgp = torch.empty(T, C, device=dev, dtype=dtype)
    dbias = torch.zeros(n, device=dev)
    L.check(L.load().progen_sgu_gate_bwd(ds.data_ptr(), C, a.data_ptr(), 2 * C, gp.data_ptr(), C, bias.data_ptr(), da.data_ptr(),
                                         2 * C, dgp.data_ptr(), C, dbias.data_ptr(), L.dt(a), T, C, n, L.stream()))
    t2 = 1e-5 if dtype == torch.float32 else 5e-2
    assert (da[:, :C].double() - xs.grad).abs().max().item() < t2
    assert (dgp.double() - gpd.grad).abs().max().item() < t2
    assert (dbias.double() - bd.grad).abs().max().item() < (1e-4 if dtype == torch.float32 else 0.3)
    # gelu backward
    u = torch.randn(T, C, generator=g, device=dev).to(dtype)
    d2 = ds.clone()
    L.check(L.load().progen_gelu_bwd(d2.data_ptr(), u.data_ptr(), L.dt(u), T * C, L.stream()))
    assert (d2.double() - ds.double() * gelu_grad(u.double())).abs().max().item() < t2


def attn_ref(qkv, B, n, w, h, dh):
    """Reference-style windowed attention (progen.py:88-102) on already-rotated q|k|v, float64."""
    T = B * n
    q, k, v = qkv.view(B, n, 3, h, dh).permute(2, 0, 3, 1, 4)           # (B, h, n, dh)
    W = n // w
    q, k, v = (t.reshape(B, h, W, w, dh) for t in (q, k, v))
    k, v = (torch.cat((torch.zeros_like(t[:, :, :1]), t), dim=2) for t in (k, v))
    k, v = (torch.cat((t[:, :, :-1], t[:, :, 1:]), dim=3) for t in (k, v))
    sim = torch.einsum('bhwid,bhwjd->bhwij', q, k) * dh ** -0.5
    mask = torch.tril(torch.ones(w, 2 * w, dtype=torch.bool, device=qkv.device), w)
    sim = torch.where(mask, sim, torch.full_like(sim, -1e10))
    attn = torch.softmax(sim, -1)
    o = torch.einsum('bhwij,bhwjd->bhwid', attn, v)
    return o.reshape(B, h, n, dh).transpose(1, 2).reshape(T, h * dh)


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('cfg', [(2, 32, 8, 2, 32), (1, 128, 64, 2, 64), (2, 48, 48, 3, 16)])
def test_local_attn_simt_fwd_bwd(dtype, cfg):
    L = _L()
    B, n, w, h, dh = cfg
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(n)
    T, I = B * n, h * dh
    qkv = torch.randn(T, 3 * I, generator=g, device=dev).to(dtype)
    out = torch.empty(T, I, device=dev, dtype=dtype)
    lse = torch.empty(T, h, device=dev)
    L.check(L.load().progen_local_attn_fwd_simt(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), L.dt(qkv), B, n, w, h, dh, L.stream()))
    qd = qkv.double().requires_grad_(True)
    ref = attn_ref(qd, B, n, w, h, dh)
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert (out.double() - ref).abs().max().item() < tol
    dout = torch.randn(T, I, generator=g, device=dev).to(dtype)
    ref.backward(dout.double())
    dqkv = torch.empty_like(qkv)
    delta = torch.empty(T, h, device=dev)
    L.check(L.load().progen_local_attn_bwd_simt(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
                                                delta.data_ptr(), L.dt(qkv), B, n, w, h, dh, L.stream()))
    tol = 2e-5 if dtype == torch.float32 else 5e-2
    assert (dqkv.double() - qd.grad).abs().max().item() < tol * max(1.0, qd.grad.abs().max().item())


def test_optimizer_chain_matches_oracle():
    L = _L()
    from oracle import progen_ref as O
    dev = 'cuda'
    rng = np.random.default_rng(0)
    params = {'a': {'w': rng.standard_normal((40, 24)).astype(np.float32)},           # ndim > 1: decayed
              'b': {'b': rng.standard_normal(64).astype(np.float32)}}                 # ndim == 1: not decayed
    n_decay, n = 40 * 24, 40 * 24 + 64
    p = torch.tensor(np.concatenate([params['a']['w'].ravel(), params['b']['b']]), device=dev)
    p_lp = torch.zeros(n, device=dev, dtype=torch.bfloat16)
    m, v, acc = (torch.zeros(n, device=dev) for _ in range(3))
    ws = torch.empty(L.load().progen_optim_workspace_floats(), device=dev)
    gn = torch.empty(1, device=dev)
    state = torch.zeros(4, dtype=torch.int64, device=dev)     # AdamDevState: the kernel counts the steps
    st = O.optim_init(params, every=4)
    cur = params
    for step in range(1, 10):
        grads = {'a': {'w': rng.standard_normal((40, 24)) * (3.0 if step % 2 else 0.01)},
                 'b': {'b': rng.standard_normal(64) * (3.0 if step % 2 else 0.01)}}
        gflat = torch.tensor(np.concatenate([grads['a']['w'].ravel(), grads['b']['b']]).astype(np.float32), device=dev)
        L.check(L.load().progen_grad_sqnorm(gflat.data_ptr(), n, ws.data_ptr(), gn.data_ptr(), L.stream()))
        L.check(L.load().progen_adamw_step(p.data_ptr(), p_lp.data_ptr(), gflat.data_ptr(), m.data_ptr(), v.data_ptr(), acc.data_ptr(),
                                           n, n_decay, gn.data_ptr(), 2e-4, 0.9, 0.999, 1e-8, 1e-3, 0.5, 4, state.data_ptr(),
                                           L.stream()))
        g32 = {k: {kk: vv.astype(np.float32) for kk, vv in d.items()} for k, d in grads.items()}
        cur, gnorm = O.optim_step(cur, g32, st)
        ref = np.concatenate([cur['a']['w'].ravel(), cur['b']['b']])
        assert abs(math.sqrt(gn.item()) - gnorm) < 1e-4 * gnorm
        assert np.abs(p.cpu().numpy() - ref).max() < 2e-6
    assert (p_lp.float() - p).abs().max().item() < 0.02
