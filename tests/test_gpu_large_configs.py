"""Config 3 (d1024 h16 w512 n2048) and config 4 (d1536 h8x64 w256 n4096) of bench.py at their own widths and sequence
lengths, against float64.

Two layers:
  * the bf16 engine's loss, row-0 logits and every gradient of a depth-3 stack of each config (one GLU layer and the two
    gMLP layers; depth only repeats these layers), by the three-way method and bounds of
    test_gpu_model.py::test_bf16_parity_at_benchmarked_shapes, with the float64 oracle and its bf16 emulation on the GPU;
  * every kernel those stacks run at the shapes the benchmarked batch gives them (T = 16384 token rows), each against a
    float64 evaluation of the same operands: LayerNorm forward / backward (including the row-kernel widths above the
    streaming kernel's 2048), every GEMM of a GLU and a gMLP layer with its epilogue and the engine's split-K, and the
    attention forward (output and log-sum-exp) and backward.

Bounds are those of the existing kernel tests, quoted where they are used."""
import json
import time

import pytest
import torch

from gemm_cases import run_case
from test_gpu_attn_tc import check_bwd as attn_check_bwd, check_fwd as attn_check_fwd
from test_gpu_elementwise import ln_ref, shift_ref
from test_gpu_gemm_tc import BF16_OUT_TOL, F32_OUT_TOL
from test_gpu_model import bf16_three_way

pytestmark = pytest.mark.gpu

# bench.py's configurations (per-GPU batch: 8 sequences of 2048, 4 sequences of 4096), at depth 3 = 1 GLU + 2 gMLP layers
CONFIGS = {
    'cfg3': dict(kwargs=dict(num_tokens=256, dim=1024, seq_len=2048, depth=3, heads=16, dim_head=64, window_size=512,
                             global_mlp_depth=2, ff_glu=True), batch=8),
    'cfg4': dict(kwargs=dict(num_tokens=256, dim=1536, seq_len=4096, depth=3, heads=8, dim_head=64, window_size=256,
                             global_mlp_depth=2, ff_glu=True), batch=4),
}


def _no_tf32():
    # `emu` must be the ideal bf16-operand / fp32-accumulate evaluation: its fp32 matmuls may not run as TF32
    assert torch.get_float32_matmul_precision() == 'highest', torch.get_float32_matmul_precision()
    assert torch.backends.cuda.matmul.allow_tf32 is False


# ------------------------------------------------------------------------------------------------ model-level parity
@pytest.mark.parametrize('case', ['cfg3_stack', 'cfg4_stack'])
def test_bf16_parity_at_large_config_stacks(case):
    """ref (float64 oracle) / emu (fp32 oracle, bf16 operands) / cuda (ProGen mixed_precision) at B = 2 sequences of the
    config's own length, one padded after n/2.  ref and emu run on the GPU: several TFLOP of float64 autograd."""
    _no_tf32()
    kwargs = CONFIGS[case.split('_')[0]]['kwargs']
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    try:
        bf16_three_way(case, kwargs, 2, device='cuda')
    finally:
        torch.cuda.synchronize()
        print(json.dumps(dict(case=case, peak_device_memory_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                              device_memory_gib=round(torch.cuda.get_device_properties(0).total_memory / 2 ** 30, 2),
                              wall_s=round(time.perf_counter() - t0, 1))))


# ------------------------------------------------------------------------------------------------ LayerNorm
def _L():
    from progen_b200 import lib as L
    L.require_device()
    return L


@pytest.mark.parametrize('C,B,n', [(3072, 2, 4096), (2048, 2, 2048)])
def test_ln_sgu_gate_strided_nonresidual(C, B, n):
    """The gMLP gate norm: bf16 input and input gradient as the second half of a 2C-wide buffer, bf16 output, no residual.
    C = 3072 (config 4) is wider than the streaming kernel's 2048 and runs on the row-per-warp kernel (NCH = 32);
    C = 2048 (config 3) is the streaming kernel's widest instantiation (16 chunks of 128, 4-row stages).
    Bounds: test_ln_strided_act_input (row kernel), test_ln_bwd_stream_path_strided_nonresidual (streaming kernel)."""
    L = _L()
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(C + n)
    T = B * n
    a = torch.randn(T, 2 * C, generator=g, device=dev).bfloat16()
    scale = torch.randn(C, generator=g, device=dev)
    y = torch.empty(T, C, device=dev, dtype=torch.bfloat16)
    mean = torch.empty(T, device=dev)
    rstd = torch.empty(T, device=dev)
    gate = a[:, C:]
    L.check(L.load().progen_ln_shift_fwd(gate.data_ptr(), 2 * C, L.BF16, scale.data_ptr(), y.data_ptr(), C, L.BF16,
                                         mean.data_ptr(), rstd.data_ptr(), T, C, n, 0, L.stream()))
    xd = gate.double().requires_grad_(True)
    sd = scale.double().requires_grad_(True)
    ref = ln_ref(xd, sd)
    assert (y.double() - ref).abs().max().item() < 2e-2 * ref.abs().max().item()
    dy = torch.randn(T, C, generator=g, device=dev).bfloat16()
    da = torch.zeros(T, 2 * C, device=dev, dtype=torch.bfloat16)
    dscale = torch.zeros(C, device=dev)
    L.check(L.load().progen_ln_shift_bwd(dy.data_ptr(), C, L.BF16, gate.data_ptr(), 2 * C, L.BF16, scale.data_ptr(),
                                         mean.data_ptr(), rstd.data_ptr(), 0, da[:, C:].data_ptr(), 2 * C, dscale.data_ptr(), 0,
                                         T, C, n, 0, 0, L.stream()))
    ref.backward(dy.double())
    assert (da[:, C:].double() - xd.grad).abs().max().item() < 2e-2 * xd.grad.abs().max().item()
    assert da[:, :C].abs().max().item() == 0
    ds_tol = 1e-3 if C > 2048 else 2e-3
    assert (dscale.double() - sd.grad).abs().max().item() < ds_tol * sd.grad.abs().max().item()


@pytest.mark.parametrize('d,B,n', [
    (1536, 4, 4096),       # config 4's residual LayerNorms: streaming kernel <12, ..., 4>
    (2048, 2, 2048),       # streaming kernel <16, ..., 4>, fp32-input residual form
    (3072, 2, 2048),       # row-per-warp kernel, NCH = 32
    (4096, 2, 2048),       # the widest d progen_ln_shift_bwd accepts (row-per-warp kernel, NCH = 32)
])
def test_ln_residual_shift_wide(d, B, n):
    """fp32 residual stream in, bf16 LN output, token shift; backward accumulates into the fp32 residual gradient with a
    bf16 copy and the column sums.  Bounds: test_ln_bwd_stream_path_residual."""
    L = _L()
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(d + n)
    T = B * n
    act = torch.bfloat16
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
    assert (y.double() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item())
    dy = torch.randn(T, d, generator=g, device=dev).to(act)
    dres0 = torch.randn(T, d, generator=g, device=dev)
    dres = dres0.clone()
    dres_lp = torch.full((T, d), float('nan'), device=dev, dtype=act)
    dscale = torch.zeros(d, device=dev)
    csum = torch.zeros(d, device=dev)
    L.check(L.load().progen_ln_shift_bwd(dy.data_ptr(), d, L.dt(dy), x.data_ptr(), d, L.F32, scale.data_ptr(), mean.data_ptr(),
                                         rstd.data_ptr(), dres.data_ptr(), dres_lp.data_ptr(), d, dscale.data_ptr(),
                                         csum.data_ptr(), T, d, n, 1, 1, L.stream()))
    ref.backward(dy.double())
    gs = max(1.0, xd.grad.abs().max().item())
    assert (dres.double() - (dres0.double() + xd.grad)).abs().max().item() < 1e-4 * gs
    assert (dscale.double() - sd.grad).abs().max().item() < 1e-3 * max(1.0, sd.grad.abs().max().item())
    assert (dres_lp.double() - dres.double()).abs().max().item() <= 0.06
    cs_ref = dres.double().sum(0)
    assert (csum.double() - cs_ref).abs().max().item() < 1e-3 * max(1.0, cs_ref.abs().max().item())


# ------------------------------------------------------------------------------------------------ GEMM
def _gemm_shapes(name):
    """{id: (M, N, K, a_mn, b_mn, epi, wgrad (K_in, N_out) or None)} of every GEMM of one GLU and one gMLP layer of config
    `name` (the spatial GEMMs apart: test_sgu_spatial_gemms), as Engine._forward_device / _backward_body issue them at
    the benchmarked batch"""
    from progen_b200 import lib as L
    c = CONFIGS[name]
    kw = c['kwargs']
    d, I, hid = kw['dim'], kw['heads'] * kw['dim_head'], 4 * kw['dim']
    half, T = hid // 2, c['batch'] * kw['seq_len']
    fwd = lambda N, K, epi: (T, N, K, False, True, epi, None)
    dgrad = lambda N, K, epi=L.EPI_STORE: (T, N, K, False, False, epi, None)
    wgrad = lambda K_in, N_out: (K_in, N_out, T, True, True, L.EPI_ACCUM, (K_in, N_out))
    return {
        # attention block (both layer kinds)
        'qkv_rotary': fwd(3 * I, d, L.EPI_ROTARY), 'attn_out_residual': fwd(d, I, L.EPI_RESIDUAL),
        'attn_out_dgrad': dgrad(I, d), 'attn_out_wgrad': wgrad(I, d),
        'qkv_dgrad': dgrad(d, 3 * I), 'qkv_wgrad': wgrad(d, 3 * I),
        # GLU feed-forward
        'glu_in': fwd(2 * hid, d, L.EPI_GLU), 'glu_out_residual': fwd(d, hid, L.EPI_RESIDUAL),
        'glu_out_dgrad_glu_bwd': dgrad(hid, d, L.EPI_GLU_BWD), 'glu_out_wgrad': wgrad(hid, d),
        'glu_in_dgrad': dgrad(d, 2 * hid), 'glu_in_wgrad': wgrad(d, 2 * hid),
        # gMLP feed-forward
        'sgu_in_gelu': fwd(hid, d, L.EPI_GELU), 'sgu_proj': fwd(half, half, L.EPI_STORE),
        'sgu_out_residual': fwd(d, half, L.EPI_RESIDUAL), 'sgu_out_dgrad': dgrad(half, d),
        'sgu_out_wgrad': wgrad(half, d), 'sgu_proj_dgrad': dgrad(half, half), 'sgu_proj_wgrad': wgrad(half, half),
        'sgu_in_dgrad': dgrad(d, hid), 'sgu_in_wgrad': wgrad(d, hid),
        # the plain-GELU feed-forward's (ff_glu=False) dgrad epilogue at this width
        'gelu_out_dgrad_gelu_bwd': dgrad(hid, d, L.EPI_GELU_BWD),
    }


_SPLITS = {}


def _wgrad_split(name, K_in, N_out):
    """Engine.wgrad_split of an engine built for config `name` at its benchmarked batch (the split depends on the number
    of token rows and the SM count)"""
    if name not in _SPLITS:
        from progen_b200.engine import Engine
        from oracle import progen_ref as O
        c = CONFIGS[name]
        eng = Engine(O.make_config(**c['kwargs']), mixed_precision=True)
        eng.ensure_batch(c['batch'])
        _SPLITS[name] = {s[6]: eng.wgrad_split(*s[6]) for s in _gemm_shapes(name).values() if s[6]}
        del eng
        torch.cuda.empty_cache()
    return _SPLITS[name][(K_in, N_out)]


@pytest.mark.parametrize('name,gemm', [(n, g) for n in CONFIGS for g in _gemm_shapes(n)])
def test_gemm_at_config_shapes(name, gemm):
    """wgmma GEMM + epilogue against float64 of the same bf16 operands (gemm_cases.run_case).  Bounds: test_gpu_gemm_tc.py
    (one bf16 ulp for bf16 outputs, F32_OUT_TOL for the fp32 residual stream, 1e-3 for split-K weight gradients as in
    test_tc_gemm_split_k_wgrad)."""
    from progen_b200 import lib as L
    M, N, K, a_mn, b_mn, epi, wgrad = _gemm_shapes(name)[gemm]
    split = _wgrad_split(name, *wgrad) if wgrad else 1
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, M, N, K, a_mn, b_mn, epi, seed=M + N + K + epi, split_k=split,
                          seq_len=CONFIGS[name]['kwargs']['seq_len'], dim_head=64)
    if epi == L.EPI_ACCUM:
        tol = 1e-3 if split > 1 else F32_OUT_TOL
    else:
        tol = F32_OUT_TOL if epi == L.EPI_RESIDUAL else BF16_OUT_TOL
    assert err <= tol * max(1.0, scale), (split, err, scale)


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_sgu_spatial_gemms(name):
    """The gMLP spatial GEMMs at the config's batch: gate_b = tril(W) @ gn_b (causal 1), d gn_b = tril(W)^T @ dGp_b
    (causal 2), and d W = tril(sum_b dGp_b gn_b^T) (batch reduction into the fp32 gradient, upper triangle untouched).
    Bounds: test_tc_batched_causal_and_reduce."""
    from progen_b200 import lib as L
    c = CONFIGS[name]
    B, n, C = c['batch'], c['kwargs']['seq_len'], 2 * c['kwargs']['dim']
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(n + C)
    Wm = torch.tril(torch.randn(n, n, generator=g, device=dev) * n ** -0.5).bfloat16()
    X = torch.randn(B * n, C, generator=g, device=dev).bfloat16()
    Xd = X.view(B, n, C).double()
    out = torch.empty(B * n, C, device=dev, dtype=torch.bfloat16)
    L.gemm(M=n, N=C, K=n, A=Wm, lda=n, B=X, ldb=C, b_mn=True, out=out, ldo=C, backend=L.BACKEND_TC, in_dtype=L.BF16,
           out_dtype=L.BF16, batch=B, b_batch_rows=n, d_batch_rows=n, causal=1)
    ref = torch.einsum('mk,bkc->bmc', Wm.double(), Xd).reshape(B * n, C)
    assert (out.double() - ref).abs().max().item() <= BF16_OUT_TOL * ref.abs().max().item()
    L.gemm(M=n, N=C, K=n, A=Wm, lda=n, a_mn=True, B=X, ldb=C, b_mn=True, out=out, ldo=C, backend=L.BACKEND_TC,
           in_dtype=L.BF16, out_dtype=L.BF16, batch=B, b_batch_rows=n, d_batch_rows=n, causal=2)
    ref = torch.einsum('km,bkc->bmc', Wm.double(), Xd).reshape(B * n, C)
    assert (out.double() - ref).abs().max().item() <= BF16_OUT_TOL * ref.abs().max().item()
    del ref
    G = torch.randn(B * n, C, generator=g, device=dev).bfloat16()
    dW = torch.zeros(n, n, device=dev)
    L.gemm(M=n, N=n, K=C, A=G, lda=C, B=X, ldb=C, out=dW, ldo=n, backend=L.BACKEND_TC, in_dtype=L.BF16,
           epi=L.EPI_ACCUM, batch=B, a_batch_rows=n, b_batch_rows=n, batch_reduce=True, atomic=True, tril=True, tril_rows=n)
    ref = torch.tril(torch.einsum('bmc,bkc->mk', G.view(B, n, C).double(), Xd))
    assert (dW.double() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


# ------------------------------------------------------------------------------------------------ attention
ATTN = [pytest.param((2, 4096, 256, 8), id='cfg4'), pytest.param((2, 2048, 512, 16), id='cfg3')]      # (B, n, w, h)


@pytest.mark.parametrize('cfg', ATTN)
def test_attn_fwd_and_lse_vs_float64(cfg):
    """tensor-core forward: test_local_attn_tc_fwd's checks, and the log-sum-exp against the float64 log-sum-exp of the
    scaled, masked scores (window 0 includes its w zero look-back keys) with test_local_attn_tc_fwd's lse bound"""
    qkv, out, lse = attn_check_fwd(cfg)
    B, n, w, h = cfg
    dh = 64
    q, k, _ = qkv.double().view(B, n, 3, h, dh).permute(2, 0, 3, 1, 4)
    W = n // w
    q, k = q.reshape(B, h, W, w, dh), k.reshape(B, h, W, w, dh)
    k = torch.cat((torch.zeros_like(k[:, :, :1]), k), dim=2)
    k = torch.cat((k[:, :, :-1], k[:, :, 1:]), dim=3)
    sim = torch.einsum('bhwid,bhwjd->bhwij', q, k) * dh ** -0.5
    mask = torch.tril(torch.ones(w, 2 * w, dtype=torch.bool, device=qkv.device), w)
    ref = torch.logsumexp(sim.masked_fill(~mask, float('-inf')), -1)              # (B, h, W, w)
    ref = ref.reshape(B, h, n).transpose(1, 2).reshape(B * n, h)
    err = (lse.double() - ref).abs().max().item()
    assert err < 2e-3, err


@pytest.mark.parametrize('cfg', ATTN)
@pytest.mark.parametrize('fused_rotary', [False, True])
def test_attn_bwd(cfg, fused_rotary):
    """tensor-core backward with and without the fused rotary backward: test_local_attn_tc_bwd's checks at these shapes"""
    attn_check_bwd(cfg, fused_rotary)
