"""Tensor-core local attention (attn_wgmma.cu: forward, dQ + dK/dV) against a torch float64 reference of reference
progen.py:88-102 computed from the same bf16 q|k|v, and against the exact-fp32 CUDA-core kernel, forward and backward,
including window 0's zero look-back keys (quirk Q1).  The shapes include windows that are multiples of 64 but not of
128 (64, 192, 320)."""
import pytest
import torch

from test_gpu_elementwise import attn_ref

pytestmark = pytest.mark.gpu

SHAPES = [(2, 256, 128, 2), (1, 512, 256, 3), (2, 192, 64, 2), (1, 1024, 256, 8), (3, 128, 128, 1), (2, 1024, 512, 2),
          (5, 512, 256, 8), (4, 256, 64, 4), (2, 384, 192, 2), (1, 640, 320, 3)]


def _qkv(B, n, h, dh, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randn(B * n, 3 * h * dh, generator=g, device='cuda') * 1.5).bfloat16(), g


@pytest.mark.parametrize('cfg', SHAPES)
def test_local_attn_tc_fwd(cfg):
    """forward vs the float64 reference, and output and log-sum-exp vs the fp32 simt kernel on the same bf16 input"""
    check_fwd(cfg)


def check_fwd(cfg):
    """the checks of test_local_attn_tc_fwd at shape cfg = (B, n, w, h); returns (qkv, out, lse) for further checks"""
    from progen_b200 import lib as L
    L.require_device()
    B, n, w, h = cfg
    dh = 64
    T, I = B * n, h * dh
    qkv, _ = _qkv(B, n, h, dh, 7 * n + w)
    out = torch.full((T, I), float('nan'), device='cuda', dtype=torch.bfloat16)
    lse = torch.full((T, h), float('nan'), device='cuda')
    L.check(L.load().progen_local_attn_fwd_tc(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, w, h, dh, L.stream()))
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    ref = attn_ref(qkv.double(), B, n, w, h, dh)
    err = (out.double() - ref).abs().max().item()
    assert err < 2e-2, err
    out2 = torch.empty_like(out)
    lse2 = torch.empty_like(lse)
    L.check(L.load().progen_local_attn_fwd_simt(qkv.data_ptr(), out2.data_ptr(), lse2.data_ptr(), L.BF16, B, n, w, h, dh, L.stream()))
    assert (lse - lse2).abs().max().item() < 2e-3
    assert (out.float() - out2.float()).abs().max().item() < 2e-2
    return qkv, out, lse


@pytest.mark.parametrize('cfg', SHAPES)
@pytest.mark.parametrize('fused_rotary', [False, True])
def test_local_attn_tc_bwd(cfg, fused_rotary):
    """backward on the tensor-core forward's out and lse vs torch float64 autograd of the reference attention on the same
    bf16 q|k|v; with fused_rotary, also vs the unfused kernel's gradient with the rotary backward applied in torch"""
    check_bwd(cfg, fused_rotary)


def check_bwd(cfg, fused_rotary):
    """the checks of test_local_attn_tc_bwd at shape cfg = (B, n, w, h)"""
    from progen_b200 import lib as L
    from gemm_cases import rotary_tables
    L.require_device()
    B, n, w, h = cfg
    dh = 64
    dev = 'cuda'
    T, I = B * n, h * dh
    qkv, g = _qkv(B, n, h, dh, 3 * n + w)
    out = torch.empty(T, I, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(T, h, device=dev)
    L.check(L.load().progen_local_attn_fwd_tc(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, w, h, dh, L.stream()))
    dout = torch.randn(T, I, generator=g, device=dev).bfloat16()
    qd = qkv.double().requires_grad_(True)
    attn_ref(qd, B, n, w, h, dh).backward(dout.double())
    grad = qd.grad
    sin, cos = rotary_tables(n, dh, dev)
    pos = torch.arange(T, device=dev) % n
    s_ = sin.double()[pos].repeat(1, 3 * h)
    c_ = cos.double()[pos].repeat(1, 3 * h)

    def rotary_bwd(x):
        x0, x1 = x[:, 0::2], x[:, 1::2]
        return torch.stack((x0 * c_ + x1 * s_, x1 * c_ - x0 * s_), dim=-1).flatten(-2)

    def bwd(rot):
        dqkv = torch.full_like(qkv, float('nan'))
        delta = torch.full((T, h), float('nan'), device=dev)
        L.check(L.load().progen_local_attn_bwd_tc(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(),
                                                  delta.data_ptr(), sin.data_ptr() if rot else 0, cos.data_ptr() if rot else 0,
                                                  B, n, w, h, dh, L.stream()))
        torch.cuda.synchronize()
        assert torch.isfinite(dqkv.float()).all() and torch.isfinite(delta).all()
        return dqkv.double(), delta

    dqkv, delta = bwd(fused_rotary)
    if fused_rotary:
        grad = rotary_bwd(grad)
    dref = (out.double().view(T, h, dh) * dout.double().view(T, h, dh)).sum(-1)
    assert (delta.double() - dref).abs().max().item() < 1e-2 * max(1.0, dref.abs().max().item())
    gerr = (dqkv - grad).abs().max().item()
    assert gerr < 4e-2 * max(1.0, grad.abs().max().item()), (gerr, grad.abs().max().item())
    for part, name in enumerate(('dq', 'dk', 'dv')):
        a_ = dqkv[:, part * I:(part + 1) * I]
        r_ = grad[:, part * I:(part + 1) * I]
        rel = (a_ - r_).norm().item() / r_.norm().item()
        assert rel < 2e-2, (name, rel)
        assert (a_ - r_).abs().max().item() < 5e-2 * max(1.0, r_.abs().max().item()), name
    if fused_rotary:
        # fused rotary backward == the rotary backward applied in torch to the kernel's un-fused result
        expect = rotary_bwd(bwd(False)[0])
        assert (dqkv - expect).abs().max().item() < 3e-2 * max(1.0, expect.abs().max().item())
