"""The wgmma GEMM's split epilogue (global reads issued for a whole pass before its items are finished) and the column
sums the GLU / GELU backward epilogues add into the proj_in bias gradient."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


@pytest.mark.parametrize('M,N,K', [(32832, 544, 256),      # ~10 tiles per CTA, a 64-row tail and a 32-column tail
                                   (200, 160, 128)])       # tails in both passes of one tile row
@pytest.mark.parametrize('inplace', [False, True])
def test_residual_epilogue_is_store_plus_residual_bitwise(M, N, K, inplace):
    """out = aux + (acc + bias): bit for bit the fp32 EPI_STORE output (with bias) of the same GEMM plus aux in torch"""
    from progen_b200 import lib as L
    g = _gen(1)
    x = torch.randn(M, K, generator=g, device='cuda').bfloat16()
    w = (torch.randn(K, N, generator=g, device='cuda') * K ** -0.5).bfloat16()
    bias = torch.randn(N, generator=g, device='cuda')
    res = torch.randn(M, N, generator=g, device='cuda')
    kw = dict(M=M, N=N, K=K, A=x, lda=K, B=w, ldb=N, b_mn=True, ldo=N, backend=L.BACKEND_TC, in_dtype=L.BF16,
              out_dtype=L.F32, bias=bias)
    stored = torch.full((M, N), float('nan'), device='cuda')
    L.gemm(out=stored, epi=L.EPI_STORE, **kw)
    if inplace:
        out = res.clone()
        L.gemm(out=out, epi=L.EPI_RESIDUAL, **kw)
    else:
        out = torch.full((M, N), float('nan'), device='cuda')
        L.gemm(out=out, epi=L.EPI_RESIDUAL, aux=res, ldaux=N, **kw)
    torch.cuda.synchronize()
    assert torch.equal(out, res + stored)


def _bwd_case(epi, M, N, K, seed):
    """dgrad + GLU / GELU backward operands: dy [M, K], w [N, K] (K-major), saved pre-activation aux"""
    from progen_b200 import lib as L
    g = _gen(seed)
    width = 2 * N if epi == L.EPI_GLU_BWD else N
    dy = torch.randn(M, K, generator=g, device='cuda').bfloat16()
    w = (torch.randn(N, K, generator=g, device='cuda') * K ** -0.5).bfloat16()
    aux = (2 * torch.randn(M, width, generator=g, device='cuda')).bfloat16()
    return dy, w, aux, width


def _bwd(epi, dy, w, aux, width, M, N, K, colsum=None, backend=None, dtype=torch.bfloat16):
    from progen_b200 import lib as L
    du = torch.full((M, width), float('nan'), device='cuda', dtype=dtype)
    dt = L.BF16 if dtype == torch.bfloat16 else L.F32
    L.gemm(M=M, N=N, K=K, A=dy, lda=K, B=w, ldb=K, out=du, ldo=width, epi=epi, aux=aux, ldaux=width,
           backend=L.BACKEND_TC if backend is None else backend, in_dtype=dt, out_dtype=dt, colsum=colsum)
    return du


@pytest.mark.parametrize('epi_name', ['EPI_GLU_BWD', 'EPI_GELU_BWD'])
@pytest.mark.parametrize('M,N,K', [(8256, 2080, 512),     # many tiles per CTA, a 64-row tail, a 32-column tail
                                   (100, 96, 64)])        # one partial tile
def test_backward_colsum(epi_name, M, N, K):
    from progen_b200 import lib as L
    epi = getattr(L, epi_name)
    dy, w, aux, width = _bwd_case(epi, M, N, K, seed=2)
    plain = _bwd(epi, dy, w, aux, width, M, N, K)
    # colsum adds onto what is there; the 32 entries past the output columns must stay untouched
    base = torch.randn(width + 32, generator=_gen(3), device='cuda')
    cs = base.clone()
    fused = _bwd(epi, dy, w, aux, width, M, N, K, colsum=cs)
    torch.cuda.synchronize()
    assert torch.equal(fused, plain), 'the column sum changed du'
    assert not torch.isnan(fused).any()
    assert torch.equal(cs[width:], base[width:]), 'columns outside N were written'
    du = fused.double()
    ref = base[:width].double() + du.sum(0)
    # any fp32 summation order of M + 1 terms: |error| <= (M + 1) u sum |terms|, u = 2^-24
    bound = (M + 1) * 2.0 ** -24 * (base[:width].double().abs() + du.abs().sum(0))
    err = (cs[:width].double() - ref).abs()
    assert (err <= bound).all(), (err.max().item(), bound.min().item())


@pytest.mark.parametrize('epi_name', ['EPI_GLU_BWD', 'EPI_GELU_BWD'])
def test_backward_colsum_simt(epi_name):
    """the fp32 CUDA-core GEMM shares the epilogue: same du with and without the column sum, and the sum itself"""
    from progen_b200 import lib as L
    epi = getattr(L, epi_name)
    M, N, K = 300, 136, 96
    dy, w, aux, width = _bwd_case(epi, M, N, K, seed=4)
    dy, w, aux = dy.float(), w.float(), aux.float()
    plain = _bwd(epi, dy, w, aux, width, M, N, K, backend=L.BACKEND_SIMT, dtype=torch.float32)
    cs = torch.zeros(width, device='cuda')
    fused = _bwd(epi, dy, w, aux, width, M, N, K, colsum=cs, backend=L.BACKEND_SIMT, dtype=torch.float32)
    torch.cuda.synchronize()
    assert torch.equal(fused, plain)
    du = fused.double()
    bound = (M + 1) * 2.0 ** -24 * du.abs().sum(0)
    assert ((cs.double() - du.sum(0)).abs() <= bound).all()


def test_colsum_only_with_backward_epilogues():
    from progen_b200 import lib as L
    x = torch.zeros(128, 64, device='cuda', dtype=torch.bfloat16)
    w = torch.zeros(128, 64, device='cuda', dtype=torch.bfloat16)
    out = torch.empty(128, 128, device='cuda', dtype=torch.bfloat16)
    cs = torch.zeros(128, device='cuda')
    with pytest.raises(L.ProgenError):
        L.gemm(M=128, N=128, K=64, A=x, lda=64, B=w, ldb=64, out=out, ldo=128, backend=L.BACKEND_TC, in_dtype=L.BF16,
               out_dtype=L.BF16, epi=L.EPI_STORE, colsum=cs)


@pytest.mark.parametrize('ff_glu', [True, False])
def test_step_proj_in_bias_grad_matches_colsum_pass(ff_glu):
    """A training step at the config-2 width (d 512, hid 2048, 8 heads of 64): the proj_in bias gradients the backward
    epilogues sum match a separate progen_colsum pass over du; every other gradient is unaffected."""
    from progen_b200 import ProGen
    from progen_b200 import lib as L
    from oracle import progen_ref as O
    kwargs = dict(num_tokens=256, dim=512, seq_len=256, depth=2, window_size=256, global_mlp_depth=0, heads=8, dim_head=64,
                  ff_glu=ff_glu)
    cfg = O.make_config(**kwargs)
    params = O.randomize_params(O.init_params(cfg, 3), 4)
    data = np.random.default_rng(5).integers(0, 256, (4, cfg['seq_len'] + 1)).astype(np.uint16)
    model = ProGen(**kwargs, mixed_precision=True)
    _, fused = model.loss_and_grad(params, data)

    eng = model.engine
    fused_dgrad = eng.dgrad_gemm

    def colsum_pass(dy, N_out, w, K_in, out, epi=L.EPI_STORE, colsum=None, **kw):
        fused_dgrad(dy, N_out, w, K_in, out, epi=epi, **kw)
        if colsum is not None:
            eng.colsum(out, 2 * K_in if epi == L.EPI_GLU_BWD else K_in, colsum)
    eng.dgrad_gemm = colsum_pass
    try:
        _, ref = model.loss_and_grad(params, data)
    finally:
        del eng.dgrad_gemm
    checked = 0
    for m, d in ref.items():
        for k, r in d.items():
            scale = max(1e-8, np.abs(r).max())
            err = np.abs(fused[m][k] - r).max()
            assert err < 2e-4 * scale + 1e-7, (m, k, err, scale)
            if k == 'b' and m.endswith('/linear') and '/ff' in m:
                checked += 1
    assert checked == kwargs['depth']
