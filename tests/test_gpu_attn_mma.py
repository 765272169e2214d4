"""Tensor-core local attention (attn_mma.cu) against a torch float64 reference of reference progen.py:88-102 computed
from the same bf16 q|k|v, forward and backward, including window 0's zero look-back keys (quirk Q1)."""
import pytest
import torch

from test_gpu_elementwise import attn_ref

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('cfg', [(2, 256, 128, 2), (1, 512, 256, 3), (2, 192, 64, 2), (1, 1024, 256, 8), (3, 128, 128, 1)])
def test_local_attn_mma_fwd_bwd(cfg):
    from progen_b200 import lib as L
    L.require_device()
    B, n, w, h = cfg
    dh = 64
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(n + w)
    T, I = B * n, h * dh
    qkv = (torch.randn(T, 3 * I, generator=g, device=dev) * 1.5).bfloat16()
    out = torch.empty(T, I, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(T, h, device=dev)
    L.check(L.load().progen_local_attn_fwd(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, w, h, dh, L.stream()))
    qd = qkv.double().requires_grad_(True)
    ref = attn_ref(qd, B, n, w, h, dh)
    err = (out.double() - ref).abs().max().item()
    assert err < 2e-2, err
    # lse against the fp32-exact CUDA-core kernel
    out2 = torch.empty_like(out)
    lse2 = torch.empty_like(lse)
    L.check(L.load().progen_local_attn_fwd_simt(qkv.data_ptr(), out2.data_ptr(), lse2.data_ptr(), L.BF16, B, n, w, h, dh, L.stream()))
    assert (lse - lse2).abs().max().item() < 2e-3
    dout = torch.randn(T, I, generator=g, device=dev).bfloat16()
    ref.backward(dout.double())
    dqkv = torch.full_like(qkv, float('nan'))
    delta = torch.empty(T, h, device=dev)
    L.check(L.load().progen_local_attn_bwd(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
                                           delta.data_ptr(), 0, 0, B, n, w, h, dh, L.stream()))
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all()
    gerr = (dqkv.double() - qd.grad).abs().max().item()
    assert gerr < 4e-2 * max(1.0, qd.grad.abs().max().item()), (gerr, qd.grad.abs().max().item())
    # per-part relative error (dq, dk, dv)
    for part in range(3):
        a = dqkv.double()[:, part * I:(part + 1) * I]
        r = qd.grad[:, part * I:(part + 1) * I]
        rel = (a - r).norm().item() / r.norm().item()
        assert rel < 2e-2, (part, rel)
    # fused rotary backward == separate rotary_bwd kernel applied to the un-fused result
    from gemm_cases import rotary_tables
    sin, cos = rotary_tables(n, dh, dev)
    fused = torch.empty_like(qkv)
    L.check(L.load().progen_local_attn_bwd(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), fused.data_ptr(),
                                           delta.data_ptr(), sin.data_ptr(), cos.data_ptr(), B, n, w, h, dh, L.stream()))
    ref2 = torch.stack((dqkv.double()[:, 0::2], dqkv.double()[:, 1::2]), dim=-1)
    pos = torch.arange(T, device=dev) % n
    s_ = sin.double()[pos].repeat(1, 3 * h)
    c_ = cos.double()[pos].repeat(1, 3 * h)
    exp0 = ref2[..., 0] * c_ + ref2[..., 1] * s_
    exp1 = ref2[..., 1] * c_ - ref2[..., 0] * s_
    expect = torch.stack((exp0, exp1), dim=-1).flatten(-2)
    assert (fused.double() - expect).abs().max().item() < 3e-2 * max(1.0, expect.abs().max().item())


@pytest.mark.parametrize('cfg', [(2, 256, 128, 2), (1, 512, 256, 3), (1, 1024, 256, 8), (3, 128, 128, 1), (2, 1024, 512, 2),
                                 (5, 512, 256, 8)])
def test_local_attn_wgmma_fwd(cfg):
    """wgmma / TMA forward kernel (attn_wgmma.cu) vs the float64 reference and the mma.sync kernel's output and log-sum-exp."""
    from progen_b200 import lib as L
    L.require_device()
    B, n, w, h = cfg
    dh = 64
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(7 * n + w)
    T, I = B * n, h * dh
    qkv = (torch.randn(T, 3 * I, generator=g, device=dev) * 1.5).bfloat16()
    out = torch.full((T, I), float('nan'), device=dev, dtype=torch.bfloat16)
    lse = torch.full((T, h), float('nan'), device=dev)
    L.check(L.load().progen_local_attn_fwd_tc(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, w, h, dh, L.stream()))
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    ref = attn_ref(qkv.double(), B, n, w, h, dh)
    err = (out.double() - ref).abs().max().item()
    assert err < 2e-2, err
    out2 = torch.empty_like(out)
    lse2 = torch.empty_like(lse)
    L.check(L.load().progen_local_attn_fwd(qkv.data_ptr(), out2.data_ptr(), lse2.data_ptr(), B, n, w, h, dh, L.stream()))
    assert (lse - lse2).abs().max().item() < 2e-3
    assert (out.float() - out2.float()).abs().max().item() < 2e-2


@pytest.mark.parametrize('cfg', [(2, 256, 128, 2), (1, 512, 256, 3), (1, 1024, 256, 8), (3, 128, 128, 1), (2, 1024, 512, 2),
                                 (5, 512, 256, 8)])
@pytest.mark.parametrize('fused_rotary', [False, True])
def test_local_attn_wgmma_bwd(cfg, fused_rotary):
    """wgmma backward kernels (attn_wgmma.cu, dQ + dK/dV) vs torch float64 autograd of the reference attention on the same bf16 q|k|v."""
    from progen_b200 import lib as L
    from gemm_cases import rotary_tables
    L.require_device()
    B, n, w, h = cfg
    dh = 64
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(3 * n + w)
    T, I = B * n, h * dh
    qkv = (torch.randn(T, 3 * I, generator=g, device=dev) * 1.5).bfloat16()
    out = torch.empty(T, I, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(T, h, device=dev)
    L.check(L.load().progen_local_attn_fwd(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, w, h, dh, L.stream()))
    dout = torch.randn(T, I, generator=g, device=dev).bfloat16()
    qd = qkv.double().requires_grad_(True)
    attn_ref(qd, B, n, w, h, dh).backward(dout.double())
    grad = qd.grad
    sin, cos = rotary_tables(n, dh, dev)
    if fused_rotary:
        pos = torch.arange(T, device=dev) % n
        s_ = sin.double()[pos].repeat(1, 3 * h)
        c_ = cos.double()[pos].repeat(1, 3 * h)
        g0, g1 = grad[:, 0::2], grad[:, 1::2]
        grad = torch.stack((g0 * c_ + g1 * s_, g1 * c_ - g0 * s_), dim=-1).flatten(-2)
    dqkv = torch.full_like(qkv, float('nan'))
    delta = torch.full((T, h), float('nan'), device=dev)
    L.check(L.load().progen_local_attn_bwd_tc(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
                                              delta.data_ptr(), sin.data_ptr() if fused_rotary else 0,
                                              cos.data_ptr() if fused_rotary else 0, B, n, w, h, dh, L.stream()))
    torch.cuda.synchronize()
    assert torch.isfinite(dqkv.float()).all() and torch.isfinite(delta).all()
    dref = (out.double().view(T, h, dh) * dout.double().view(T, h, dh)).sum(-1)
    assert (delta.double() - dref).abs().max().item() < 1e-2 * max(1.0, dref.abs().max().item())
    for part, name in enumerate(('dq', 'dk', 'dv')):
        a_ = dqkv.double()[:, part * I:(part + 1) * I]
        r_ = grad[:, part * I:(part + 1) * I]
        rel = (a_ - r_).norm().item() / r_.norm().item()
        assert rel < 2e-2, (name, rel)
        assert (a_ - r_).abs().max().item() < 5e-2 * max(1.0, r_.abs().max().item()), name
