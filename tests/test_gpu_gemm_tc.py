"""wgmma / TMA GEMM (gemm_tc.cu): every operand-major combination and epilogue the engine uses, against a torch
float64 reference computed from the same bf16 operands (so the only differences are fp32 accumulation order and the
final rounding of bf16 outputs)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16_OUT_TOL = 1.0 / 128      # one bf16 ulp at the output scale
F32_OUT_TOL = 2e-4


def _tol(epi):
    from progen_b200 import lib as L
    return F32_OUT_TOL if epi in (L.EPI_RESIDUAL, L.EPI_ACCUM) else BF16_OUT_TOL


# (a_mn, b_mn, epi) combinations instantiated in gemm_tc.cu
COMBOS = [(False, True, 0), (False, False, 0), (True, True, 0), (False, True, 1), (False, True, 2), (False, True, 3),
          (False, True, 4), (False, False, 5), (False, False, 6), (True, True, 7), (False, False, 7)]


@pytest.mark.parametrize('a_mn,b_mn,epi', COMBOS)
@pytest.mark.parametrize('shape', [(256, 256, 128), (384, 128, 256), (200, 512, 192)])
def test_tc_gemm(a_mn, b_mn, epi, shape):
    from progen_b200 import lib as L
    from gemm_cases import run_case
    M, N, K = shape
    if a_mn and M % 8:
        M = 256
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, M, N, K, a_mn, b_mn, epi, seed=epi, seq_len=64 if epi == 1 else None)
    assert err <= _tol(epi) * max(1.0, scale), (err, scale)


def test_tc_gemm_many_tiles_and_long_k():
    """More tiles than SMs and a long K loop (the shared-memory ring wraps many times)."""
    from progen_b200 import lib as L
    from gemm_cases import run_case
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, 4096, 1536, 512, False, True, L.EPI_STORE, seed=3)
    assert err <= BF16_OUT_TOL * max(1.0, scale), (err, scale)
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, 128, 128, 8192, False, False, L.EPI_STORE, seed=4)
    assert err <= BF16_OUT_TOL * max(1.0, scale), (err, scale)


def test_tc_gemm_split_k_wgrad():
    from progen_b200 import lib as L
    from gemm_cases import run_case
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, 512, 1536, 4096, True, True, L.EPI_ACCUM, seed=5, split_k=6)
    assert err <= 1e-3 * max(1.0, scale), (err, scale)


def test_tc_batched_causal_and_reduce():
    from progen_b200 import lib as L
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(1)
    B, n, C = 3, 256, 128
    Wm = torch.tril(torch.randn(n, n, generator=g, device=dev)).bfloat16()
    X = torch.randn(B * n, C, generator=g, device=dev).bfloat16()
    out = torch.empty(B * n, C, device=dev, dtype=torch.bfloat16)
    L.gemm(M=n, N=C, K=n, A=Wm, lda=n, B=X, ldb=C, b_mn=True, out=out, ldo=C, backend=L.BACKEND_TC, in_dtype=L.BF16,
           out_dtype=L.BF16, batch=B, b_batch_rows=n, d_batch_rows=n, causal=1)
    ref = torch.einsum('mk,bkc->bmc', Wm.double(), X.view(B, n, C).double()).reshape(B * n, C)
    assert (out.double() - ref).abs().max().item() <= BF16_OUT_TOL * ref.abs().max().item()
    L.gemm(M=n, N=C, K=n, A=Wm, lda=n, a_mn=True, B=X, ldb=C, b_mn=True, out=out, ldo=C, backend=L.BACKEND_TC,
           in_dtype=L.BF16, out_dtype=L.BF16, batch=B, b_batch_rows=n, d_batch_rows=n, causal=2)
    ref = torch.einsum('km,bkc->bmc', Wm.double(), X.view(B, n, C).double()).reshape(B * n, C)
    assert (out.double() - ref).abs().max().item() <= BF16_OUT_TOL * ref.abs().max().item()
    G = torch.randn(B * n, C, generator=g, device=dev).bfloat16()
    dW = torch.zeros(n, n, device=dev)
    L.gemm(M=n, N=n, K=C, A=G, lda=C, B=X, ldb=C, out=dW, ldo=n, backend=L.BACKEND_TC, in_dtype=L.BF16,
           epi=L.EPI_ACCUM, batch=B, a_batch_rows=n, b_batch_rows=n, batch_reduce=True, atomic=True, tril=True, tril_rows=n)
    ref = torch.tril(torch.einsum('bmc,bkc->mk', G.view(B, n, C).double(), X.view(B, n, C).double()))
    assert (dW.double() - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


def test_tc_gemm_rotary_dim_head_64_cached_tables():
    """dim_head 64 rotary epilogue: several heads per tile, several sequences per tile's rows, and a row tail."""
    from progen_b200 import lib as L
    from gemm_cases import run_case
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, 512, 384, 128, False, True, L.EPI_ROTARY, seed=11, seq_len=128, dim_head=64)
    assert err <= BF16_OUT_TOL * max(1.0, scale), (err, scale)
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, 200, 256, 64, False, True, L.EPI_ROTARY, seed=12, seq_len=64, dim_head=64)
    assert err <= BF16_OUT_TOL * max(1.0, scale), (err, scale)


@pytest.mark.parametrize('b_mn', [False, True])
@pytest.mark.parametrize('N', [160, 224])
def test_tc_gemm_column_tail(N, b_mn):
    """N not a multiple of the 128-column tile: the last tile's TMA boxes are partly (K-major B) or wholly (MN-major B)
    outside the matrix and the epilogue skips the columns past N."""
    from progen_b200 import lib as L
    from gemm_cases import run_case
    for epi in (L.EPI_STORE, L.EPI_ACCUM) if not b_mn else (L.EPI_STORE,):
        err, scale = run_case(L.BACKEND_TC, torch.bfloat16, 384, N, 128, False, b_mn, epi, seed=30 + N)
        assert err <= _tol(epi) * max(1.0, scale), (N, b_mn, epi, err, scale)


# (b_mn, epi) combinations of the activation GEMMs (K-major A)
PAIR_COMBOS = [(True, 0), (False, 0), (True, 1), (True, 2), (True, 3), (True, 4), (False, 5), (False, 6)]


@pytest.mark.parametrize('b_mn,epi', PAIR_COMBOS)
def test_tc2_pair_kernel_many_tiles_row_tail(b_mn, epi):
    """648 tiles (several waves over the SMs), a row tail that leaves the last row tile and its TMA boxes partly outside
    the matrix, four column tiles."""
    from progen_b200 import lib as L
    from gemm_cases import run_case
    M, N, K = 256 * 80 + 136, 512, 192
    err, scale = run_case(L.BACKEND_TC, torch.bfloat16, M, N, K, False, b_mn, epi, seed=20 + epi,
                          seq_len=128 if epi == 1 else None, dim_head=64)
    assert err <= _tol(epi) * max(1.0, scale), (err, scale)


def test_tc2_pair_kernel_fp32_store_and_residual_aux():
    """fp32 STORE output and the RESIDUAL epilogue reading its input from a second buffer."""
    from progen_b200 import lib as L
    from gemm_cases import run_case
    dev = 'cuda'
    g = torch.Generator(device=dev).manual_seed(7)
    M, N, K = 1024, 256, 128
    A = torch.randn(M, K, generator=g, device=dev).bfloat16()
    B = (torch.randn(K, N, generator=g, device=dev) * K ** -0.5).bfloat16()
    acc = A.double() @ B.double()
    out = torch.empty(M, N, device=dev)
    L.gemm(M=M, N=N, K=K, A=A, lda=K, B=B, ldb=N, b_mn=True, out=out, ldo=N, backend=L.BACKEND_TC, in_dtype=L.BF16, out_dtype=L.F32)
    assert (out.double() - acc).abs().max().item() <= F32_OUT_TOL * acc.abs().max().item()
    res_in = torch.randn(M, N, generator=g, device=dev)
    keep = res_in.clone()
    bias = torch.randn(N, generator=g, device=dev)
    out2 = torch.empty(M, N, device=dev)
    L.gemm(M=M, N=N, K=K, A=A, lda=K, B=B, ldb=N, b_mn=True, out=out2, ldo=N, aux=res_in, ldaux=N, bias=bias, epi=L.EPI_RESIDUAL,
           backend=L.BACKEND_TC, in_dtype=L.BF16, out_dtype=L.F32)
    ref = keep.double() + acc + bias.double()
    assert (out2.double() - ref).abs().max().item() <= F32_OUT_TOL * ref.abs().max().item()
    assert torch.equal(res_in, keep)
