"""Time the tensor-core (wgmma) attention kernels alone, forward and backward; the default shape is BASELINE config 2
(B=64, n=1024, w=256, h=8)."""
import argparse, json, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import gpu_info
from progen_b200 import lib as L
ap = argparse.ArgumentParser(description=__doc__)
ap.add_argument('--batch', type=int, default=64)
ap.add_argument('--seq-len', type=int, default=1024)
ap.add_argument('--window', type=int, default=256)
ap.add_argument('--heads', type=int, default=8)
a = ap.parse_args()
L.require_device()
B, n, w, h, dh = a.batch, a.seq_len, a.window, a.heads, 64
T, I = B * n, h * dh
qkv = torch.randn(T, 3 * I, device='cuda').bfloat16()
out = torch.empty(T, I, device='cuda', dtype=torch.bfloat16)
dout = torch.randn(T, I, device='cuda').bfloat16()
dqkv = torch.empty_like(qkv)
lse = torch.empty(T, h, device='cuda'); delta = torch.empty(T, h, device='cuda')
lib = L.load()
def fwd(): L.check(lib.progen_local_attn_fwd_tc(qkv.data_ptr(), out.data_ptr(), lse.data_ptr(), B, n, w, h, dh, L.stream()))
def bwd(): L.check(lib.progen_local_attn_bwd_tc(qkv.data_ptr(), out.data_ptr(), dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), delta.data_ptr(), 0, 0, B, n, w, h, dh, L.stream()))
def t(f, it=20):
    for _ in range(3): f()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(it): f()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / it
flops_fwd = 4.0 * I * (w + (w + 1) / 2) * T
f, b_ = t(fwd), t(bwd)
print(json.dumps(dict(shape=dict(batch=B, seq_len=n, window=w, heads=h), fwd_ms=round(f, 4), bwd_ms=round(b_, 4),
                      fwd_tflops_causal=round(flops_fwd / f / 1e9, 1), gpu=gpu_info(torch.cuda.current_device()))))
