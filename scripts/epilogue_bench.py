"""Times the wgmma GEMM's fused epilogues at the shapes of BASELINE config 2 (d=512, hid=2048, n=1024, B=64, so T=65536
rows).  The four K = 512 GEMMs share one mainloop (8 k-blocks of 128 x 128 x 64 per tile) and differ only in their
epilogues, so their time per tile shows what each epilogue costs: QKV + rotary, attention out-proj + residual, FF proj_in
+ GLU forward, FF proj_out dgrad + GLU backward; then the FF proj_out + residual GEMM (K = 2048), and the GLU backward
followed by a separate progen_colsum pass over du against the GLU backward that adds the column sums in its epilogue.

CUDA events, one JSON line per case: ms per call, tiles, tiles per CTA, us per tile, and the card's name and power limit.
Runs against a library without the fused column sum too (it then reports that case as unsupported), so that two builds
can be alternated in one session."""
import json, os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from progen_b200 import lib as L
import bench

T, D, HID, N_SEQ, DH = 65536, 512, 2048, 1024, 64
BM = BN = 128


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


def report(name, ms, M, N, K, gpu, sms, **extra):
    tiles = -(-M // BM) * -(-N // BN)
    per_cta = tiles / min(tiles, sms)
    print(json.dumps(dict(name=name, ms=round(ms, 4), M=M, N=N, K=K, tiles=tiles, tiles_per_cta=round(per_cta, 2),
                          us_per_tile=round(ms * 1e3 / per_cta, 3), gpu=gpu['name'], power_limit_w=gpu['power_limit_w'],
                          **extra)), flush=True)


def bf(*shape):
    return torch.randn(*shape, device='cuda').bfloat16()


def main():
    L.require_device()
    gpu = bench.gpu_info(torch.cuda.current_device())
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    fused = 'colsum' in dict(L.GemmDesc._fields_)
    empty = lambda *s, dt=torch.bfloat16: torch.empty(*s, device='cuda', dtype=dt)
    sin, cos = (t.float().cuda().contiguous() for t in torch.randn(2, N_SEQ, DH // 2).unbind(0))

    def fwd(N, K, epi, out, **kw):
        """out[T,N] = x[T,K] @ w[K,N] (MN-major weight), as Engine.fwd_gemm"""
        x, w = bf(T, K), bf(K, N) * K ** -0.5
        ldo = kw.pop('ldo', N)
        return lambda: L.gemm(M=T, N=N, K=K, A=x, lda=K, B=w, ldb=N, b_mn=True, out=out, ldo=ldo, backend=L.BACKEND_TC,
                              in_dtype=L.BF16, out_dtype=L.BF16, epi=epi, **kw)

    def dgrad(N, K, epi, out, **kw):
        """out[T,N] = dy[T,K] @ w[N,K]^T (K-major weight), as Engine.dgrad_gemm"""
        dy, w = bf(T, K), bf(N, K) * K ** -0.5
        ldo = kw.pop('ldo', N)
        return lambda: L.gemm(M=T, N=N, K=K, A=dy, lda=K, B=w, ldb=K, out=out, ldo=ldo, backend=L.BACKEND_TC,
                              in_dtype=L.BF16, out_dtype=L.BF16, epi=epi, **kw)

    res = torch.empty(T, D, device='cuda')
    cases = [
        ('qkv_rotary', 3 * D, D, fwd(3 * D, D, L.EPI_ROTARY, empty(T, 3 * D), rot_sin=sin, rot_cos=cos, seq_len=N_SEQ,
                                     dim_head=DH)),
        ('attn_out_residual', D, D, fwd(D, D, L.EPI_RESIDUAL, res, bias=torch.randn(D, device='cuda'),
                                        aux=torch.randn(T, D, device='cuda'), ldaux=D)),
        ('ffin_glu', 2 * HID, D, fwd(2 * HID, D, L.EPI_GLU, empty(T, HID), ldo=HID, out2=empty(T, 2 * HID), ldo2=2 * HID,
                                     bias=torch.randn(2 * HID, device='cuda'))),
        ('ffout_dgrad_glu_bwd', HID, D, dgrad(HID, D, L.EPI_GLU_BWD, empty(T, 2 * HID), ldo=2 * HID, aux=bf(T, 2 * HID),
                                              ldaux=2 * HID)),
        ('ffout_residual', D, HID, fwd(D, HID, L.EPI_RESIDUAL, res, bias=torch.randn(D, device='cuda'),
                                       aux=torch.randn(T, D, device='cuda'), ldaux=D)),
    ]
    for name, N, K, fn in cases:
        report(name, timed(fn), T, N, K, gpu, sms)

    # the proj_in bias gradient: GLU backward, then a separate column-sum pass over du [T, 2 hid] ...
    du, u, db = empty(T, 2 * HID), bf(T, 2 * HID), torch.zeros(2 * HID, device='cuda')
    glu_bwd = dgrad(HID, D, L.EPI_GLU_BWD, du, ldo=2 * HID, aux=u, ldaux=2 * HID)
    lib = L.load()

    def separate():
        glu_bwd()
        L.check(lib.progen_colsum(du.data_ptr(), 2 * HID, L.BF16, db.data_ptr(), T, 2 * HID, L.stream()), 'colsum')
    report('glu_bwd+colsum_pass', timed(separate), T, HID, D, gpu, sms)
    # ... against the column sums added by the GLU backward epilogue
    if fused:
        report('glu_bwd_fused_colsum', timed(dgrad(HID, D, L.EPI_GLU_BWD, du, ldo=2 * HID, aux=u, ldaux=2 * HID, colsum=db)),
               T, HID, D, gpu, sms)
    else:
        print(json.dumps(dict(name='glu_bwd_fused_colsum', unsupported=True, gpu=gpu['name'],
                              power_limit_w=gpu['power_limit_w'])), flush=True)


if __name__ == '__main__':
    main()
