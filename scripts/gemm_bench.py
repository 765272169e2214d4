"""Times the wgmma GEMM (gemm_tc.cu) with the fused epilogues the engine runs, at the shapes of BASELINE config 2
(d=512, hid=2048, n=1024, B=64, so T=65536 rows), and the weight-gradient GEMMs at every split-K of 1..8.  CUDA-event
timed; one JSON line per GEMM with its algorithmic bytes and FLOPs and the least time the hardware needs for them at
the data-sheet rates (the larger of FLOPs / 989 TF/s and bytes / 3.35 TB/s), then one line naming the card."""
import json, os, sys, types
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from progen_b200 import lib as L
from progen_b200.engine import Engine
import bench

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12          # NVIDIA H100 SXM data sheet (dense BF16, HBM3), not measured
T, D, HID, N_SEQ, B = 65536, 512, 2048, 1024, 64


def timed(fn):
    """mean ms per call over a window of at least ~0.2 s, after warm-up"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(5):
        fn()
    e.record(); torch.cuda.synchronize()
    iters = max(10, min(1000, int(200.0 / (s.elapsed_time(e) / 5))))
    s.record()
    for _ in range(iters):
        fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def report(name, ms, flops, nbytes, **extra):
    bound_ms = max(flops / PEAK_FLOPS, nbytes / PEAK_BYTES) * 1e3
    print(json.dumps(dict(name=name, ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1), gbytes=round(nbytes / 1e9, 3),
                          gflop=round(flops / 1e9, 1), bound_ms=round(bound_ms, 4),
                          bound='flops' if flops / PEAK_FLOPS >= nbytes / PEAK_BYTES else 'bytes',
                          time_over_bound=round(ms / bound_ms, 2), **extra)), flush=True)


def bf(*shape):
    return torch.randn(*shape, device='cuda').bfloat16()


def fwd(name, N, K, epi, out_bytes, **kw):
    """out[T,N] = x[T,K] @ w[K,N] (MN-major weight), as Engine.fwd_gemm; out_bytes: epilogue bytes per output element"""
    x, w = bf(T, K), bf(K, N) * K ** -0.5
    out = kw.pop('out')
    ms = timed(lambda: L.gemm(M=T, N=N, K=K, A=x, lda=K, B=w, ldb=N, b_mn=True, out=out, ldo=kw.get('ldo_', N),
                              backend=L.BACKEND_TC, in_dtype=L.BF16, out_dtype=L.BF16, epi=epi,
                              **{k: v for k, v in kw.items() if k != 'ldo_'}))
    report(name, ms, 2.0 * T * N * K, 2 * (T * K + K * N) + out_bytes * T * N, M=T, N=N, K=K)


def dgrad(name, N, K, epi, out_bytes, **kw):
    """out[T,N] = dy[T,K] @ w[N,K]^T (K-major weight), as Engine.dgrad_gemm"""
    dy, w = bf(T, K), bf(N, K) * K ** -0.5
    out = kw.pop('out')
    ms = timed(lambda: L.gemm(M=T, N=N, K=K, A=dy, lda=K, B=w, ldb=K, out=out, ldo=kw.get('ldo_', N), backend=L.BACKEND_TC,
                              in_dtype=L.BF16, out_dtype=L.BF16, epi=epi, **{k: v for k, v in kw.items() if k != 'ldo_'}))
    report(name, ms, 2.0 * T * N * K, 2 * (T * K + K * N) + out_bytes * T * N, M=T, N=N, K=K)


def wgrad(name, K_in, N_out, engine_split):
    """dw[K_in,N_out] += x[T,K_in]^T @ dy[T,N_out], both operands MN-major, split-K with red.global.add"""
    x, dy = bf(T, K_in), bf(T, N_out)
    dw = torch.zeros(K_in, N_out, device='cuda')
    for split in range(1, 9):
        ms = timed(lambda: L.gemm(M=K_in, N=N_out, K=T, A=x, lda=K_in, a_mn=True, B=dy, ldb=N_out, b_mn=True, out=dw,
                                  ldo=N_out, backend=L.BACKEND_TC, in_dtype=L.BF16, out_dtype=L.F32, epi=L.EPI_ACCUM,
                                  split_k=split, atomic=split > 1))
        report(name, ms, 2.0 * T * K_in * N_out, 2 * T * (K_in + N_out) + 8 * K_in * N_out, M=K_in, N=N_out, K=T,
               split_k=split, engine_split=split == engine_split)


def sgu(causal):
    """the SGU spatial mix per sequence: [n,n] lower-triangular weights times [n, hid/2] per sequence, B sequences;
    causal=1: tril(W) @ X (forward), causal=2: tril(W)^T @ dX (backward); the masked k-blocks are skipped"""
    C = HID // 2
    W, X = torch.tril(torch.randn(N_SEQ, N_SEQ, device='cuda')).bfloat16(), bf(B * N_SEQ, C)
    out = torch.empty(B * N_SEQ, C, device='cuda', dtype=torch.bfloat16)
    ms = timed(lambda: L.gemm(M=N_SEQ, N=C, K=N_SEQ, A=W, lda=N_SEQ, a_mn=causal == 2, B=X, ldb=C, b_mn=True, out=out, ldo=C,
                              backend=L.BACKEND_TC, in_dtype=L.BF16, out_dtype=L.BF16, batch=B, b_batch_rows=N_SEQ,
                              d_batch_rows=N_SEQ, causal=causal))
    flops = 2.0 * B * C * N_SEQ * (N_SEQ + 1) / 2
    report('sgu_causal%d' % causal, ms, flops, 2 * N_SEQ * N_SEQ + 2 * 2 * B * N_SEQ * C, M=N_SEQ, N=C, K=N_SEQ, batch=B)


def main():
    L.require_device()
    sin, cos = (t.float().cuda().contiguous() for t in torch.randn(2, N_SEQ, 32).unbind(0))
    bias = lambda n: torch.randn(n, device='cuda')
    empty = lambda *s, dt=torch.bfloat16: torch.empty(*s, device='cuda', dtype=dt)
    # forward
    fwd('qkv_rotary', 3 * D, D, L.EPI_ROTARY, 2, out=empty(T, 3 * D), rot_sin=sin, rot_cos=cos, seq_len=N_SEQ, dim_head=64)
    res = torch.empty(T, D, device='cuda')
    fwd('attn_out_residual', D, D, L.EPI_RESIDUAL, 8, out=res, bias=bias(D), aux=torch.randn(T, D, device='cuda'), ldaux=D)
    fwd('ffin_glu', 2 * HID, D, L.EPI_GLU, 3, out=empty(T, HID), ldo_=HID, out2=empty(T, 2 * HID), ldo2=2 * HID,
        bias=bias(2 * HID))
    fwd('ffin_gelu', HID, D, L.EPI_GELU, 4, out=empty(T, HID), out2=empty(T, HID), ldo2=HID, bias=bias(HID))
    fwd('ffout_residual', D, HID, L.EPI_RESIDUAL, 8, out=res, bias=bias(D), aux=torch.randn(T, D, device='cuda'), ldaux=D)
    # backward: dgrads (GLU backward: the saved pre-activation is read and d(pre) written, both 2 N wide)
    dgrad('ffout_dgrad_glu_bwd', HID, D, L.EPI_GLU_BWD, 8, out=empty(T, 2 * HID), ldo_=2 * HID, aux=bf(T, 2 * HID),
          ldaux=2 * HID)
    dgrad('ffout_dgrad_gelu_bwd', HID, D, L.EPI_GELU_BWD, 4, out=empty(T, HID), aux=bf(T, HID), ldaux=HID)
    dgrad('ffin_dgrad', D, 2 * HID, L.EPI_STORE, 2, out=empty(T, D))
    dgrad('qkv_dgrad', D, 3 * D, L.EPI_STORE, 2, out=empty(T, D))
    dgrad('attn_out_dgrad', D, D, L.EPI_STORE, 2, out=empty(T, D))
    # weight gradients: Engine.wgrad_split's choice is marked
    eng = types.SimpleNamespace(num_sms=torch.cuda.get_device_properties(0).multi_processor_count, T=T)
    for name, k_in, n_out in (('ffin_wgrad', D, 2 * HID), ('ffout_wgrad', HID, D), ('qkv_wgrad', D, 3 * D),
                              ('attn_out_wgrad', D, D)):
        wgrad(name, k_in, n_out, Engine.wgrad_split(eng, k_in, n_out))
    sgu(1)
    sgu(2)
    print(json.dumps(dict(gpu=bench.gpu_info(0), sms=eng.num_sms, peaks='NVIDIA H100 SXM data sheet: 989 TF/s dense BF16, '
                          '3.35 TB/s HBM3 (700 W); not measured')), flush=True)


if __name__ == '__main__':
    main()
