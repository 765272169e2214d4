"""The persistent wgmma GEMM (gemm_tc.cu) walks several tiles per CTA and hands ring stages between two consumer
warpgroups: tile lists whose tiles have different k-ranges (batched causal GEMMs of the SGU), and split-K weight
gradients with many more work units than CTAs, including K slices without k-blocks."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16_OUT_TOL = 1.0 / 128


@pytest.mark.parametrize('causal', [1, 2])
def test_tc_batched_causal_many_tiles_per_cta(causal):
    """B=16, n=1024, C=256: 256 tiles of 2 to 16 k-blocks each, more tiles than SMs"""
    from progen_b200 import lib as L
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(40 + causal)
    B, n, C = 16, 1024, 256
    Wm = (torch.tril(torch.randn(n, n, generator=g, device=dev)) * n ** -0.5).bfloat16()
    X = torch.randn(B * n, C, generator=g, device=dev).bfloat16()
    out = torch.empty(B * n, C, device=dev, dtype=torch.bfloat16)
    L.gemm(M=n, N=C, K=n, A=Wm, lda=n, a_mn=causal == 2, B=X, ldb=C, b_mn=True, out=out, ldo=C, backend=L.BACKEND_TC,
           in_dtype=L.BF16, out_dtype=L.BF16, batch=B, b_batch_rows=n, d_batch_rows=n, causal=causal)
    Wd = Wm.double() if causal == 1 else Wm.double().t()
    ref = torch.einsum('mk,bkc->bmc', Wd, X.view(B, n, C).double()).reshape(B * n, C)
    err = (out.double() - ref).abs().max().item()
    assert err <= BF16_OUT_TOL * ref.abs().max().item(), err


@pytest.mark.parametrize('shape,split', [((512, 2048, 8192), 8), ((256, 256, 640), 8)])
def test_tc_split_k_wgrad_many_units(shape, split):
    """(512, 2048, 8192) split 8: 512 work units, more than two per SM.  (256, 256, 640) split 8: 10 k-blocks in slices
    of 2, so three of the eight slices have no k-block and add zeros."""
    from progen_b200 import lib as L
    from gemm_cases import run_case
    M, N, K = shape
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, M, N, K, True, True, L.EPI_ACCUM, seed=50, split_k=split)
    assert err <= 1e-3 * max(1.0, scale), (err, scale)
