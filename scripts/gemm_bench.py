"""Micro-benchmark of the wgmma GEMM (gemm_tc.cu) against cuBLAS (torch.matmul) on the shapes of BASELINE config 2
(d=512, T=65536).  CUDA-event timed; one JSON line per shape."""
import json, sys, os, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from progen_b200 import lib as L

def bench(name, M, N, K, a_mn, b_mn, epi=L.EPI_STORE, split_k=1, iters=20):
    dev = 'cuda'
    A = torch.randn((K, M) if a_mn else (M, K), device=dev).bfloat16()
    B = torch.randn((K, N) if b_mn else (N, K), device=dev).bfloat16()
    out = torch.zeros(M, N, device=dev, dtype=torch.float32 if epi == L.EPI_ACCUM else torch.bfloat16)
    kw = dict(M=M, N=N, K=K, A=A, lda=M if a_mn else K, B=B, ldb=N if b_mn else K, out=out, ldo=N, backend=L.BACKEND_TC,
              a_mn=a_mn, b_mn=b_mn, in_dtype=L.BF16, out_dtype=L.BF16, epi=epi, split_k=split_k, atomic=split_k > 1)
    for _ in range(3):
        L.gemm(**kw)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        L.gemm(**kw)
    e.record(); torch.cuda.synchronize()
    ms = s.elapsed_time(e) / iters
    tf = 2.0 * M * N * K / ms / 1e9
    # cuBLAS reference for the same contraction
    Al = A.t() if a_mn else A
    Bl = B.t() if b_mn else B
    for _ in range(3):
        torch.matmul(Al, Bl.t())
    torch.cuda.synchronize(); s.record()
    for _ in range(iters):
        torch.matmul(Al, Bl.t())
    e.record(); torch.cuda.synchronize()
    ms2 = s.elapsed_time(e) / iters
    print(json.dumps(dict(name=name, M=M, N=N, K=K, ms=round(ms, 4), tflops=round(tf, 1), cublas_ms=round(ms2, 4),
                          cublas_tflops=round(2.0 * M * N * K / ms2 / 1e9, 1))), flush=True)

if __name__ == '__main__':
    L.require_device()
    T = 65536
    bench('qkv_fwd', T, 1536, 512, False, True)
    bench('out_fwd', T, 512, 512, False, True)
    bench('ffin_fwd', T, 4096, 512, False, True)
    bench('ffout_fwd', T, 512, 2048, False, True)
    bench('ffin_dgrad', T, 512, 4096, False, False)
    bench('ffout_dgrad', T, 2048, 512, False, False)
    bench('ffin_wgrad', 512, 4096, T, True, True, L.EPI_ACCUM, split_k=4)
    bench('qkv_wgrad', 512, 1536, T, True, True, L.EPI_ACCUM, split_k=6)
    bench('ffout_wgrad', 2048, 512, T, True, True, L.EPI_ACCUM, split_k=4)
