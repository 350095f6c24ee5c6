"""Isolated timings of the HBM-bound kernels at the OF-3B shapes (R = 8192 rows, D = 2048) against their compulsory
byte counts and the H100 SXM data-sheet HBM bandwidth."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from open_flamingo_b200 import ops

dev = "cuda"
R, D = 8192, 2048
peak = 3350.0   # GB/s: NVIDIA data-sheet HBM3 bandwidth of the H100 SXM (a peak, not a measured rate)


def timeit(fn, iters=30):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def report(name, us, nbytes):
    print(f"{name:34s} {us:8.1f} us  {nbytes/us/1e3:7.1f} GB/s  {100*nbytes/us/1e3/peak:5.1f}% of HBM peak", flush=True)


x = torch.randn(R, D, device=dev)
g = torch.randn(D, device=dev)
b = torch.randn(D, device=dev)
big = [torch.randn(R, D, device=dev) for _ in range(8)]   # rotate inputs (> L2)
outs = [torch.empty(R, D, device=dev, dtype=torch.bfloat16) for _ in range(8)]
i = [0]


def ln_fwd():
    i[0] = (i[0] + 1) % 8
    ops.layernorm_fwd(big[i[0]], g, b, out=outs[i[0]])


report("ln_fwd f32->bf16 [8192x2048]", timeit(ln_fwd), R * D * 6)
_, mean, rstd = ops.layernorm_fwd(x, g, b)
dys = [torch.randn(R, D, device=dev).to(torch.bfloat16) for _ in range(8)]
adds = [torch.randn(R, D, device=dev) for _ in range(8)]
dxs = [torch.empty(R, D, device=dev) for _ in range(8)]
dg = torch.zeros(D, device=dev)
db = torch.zeros(D, device=dev)


def ln_bwd():
    i[0] = (i[0] + 1) % 8
    ops.layernorm_bwd(dys[i[0]], big[i[0]], g, mean, rstd, dgamma=dg, dbeta=db, dx=dxs[i[0]], dx_add=adds[i[0]])


report("ln_bwd (+add, +dgamma/dbeta)", timeit(ln_bwd), R * D * (4 + 2 + 4 + 4))
gate = torch.tensor([0.3], device=dev)
dgate = torch.zeros(1, device=dev)


def gate_bwd():
    i[0] = (i[0] + 1) % 8
    ops.gate_bwd(big[i[0]], dys[i[0]], gate, dgate)


report("gate_bwd", timeit(gate_bwd), R * D * (4 + 2 + 2))
# attention cores
B, T, H = 32, 256, 8
q = torch.randn(B, T, 512, device=dev).to(torch.bfloat16)
kv = torch.randn(B, 128, 1024, device=dev).to(torch.bfloat16)
tt = torch.zeros(B, T, dtype=torch.int32, device=dev)
tt[:, 0:128] = 1
tt[:, 128:] = 2
us = timeit(lambda: ops.attn_fwd(q, kv[..., :512], kv[..., 512:], H, 0.125, mask_mode=1, text_time=tt))
report("xattn core fwd (C2)", us, (B * T * 512 * 2 + B * 128 * 1024) * 2)
qkv = torch.randn(64, 257, 3072, device=dev).to(torch.bfloat16)
us = timeit(lambda: ops.attn_fwd(qkv[..., :1024], qkv[..., 1024:2048], qkv[..., 2048:], 16, 0.125))
flops = 4 * 64 * 16 * 257 * 257 * 64
print(f"{'ViT attention fwd (64 img)':34s} {us:8.1f} us  {flops/us/1e6:7.1f} TFLOP/s", flush=True)
lq = torch.randn(32, 256, 3 * 2048, device=dev).to(torch.bfloat16)
slopes = torch.rand(16, device=dev) * 0.1
us = timeit(lambda: ops.attn_dense_fwd(lq[..., :2048], lq[..., 2048:4096], lq[..., 4096:], 16, 128, 128 ** -0.5, causal=True, slopes=slopes))
flops = 4 * 32 * 16 * 256 * 256 * 128 / 2
print(f"{'LM attention fwd (causal, hd128)':34s} {us:8.1f} us  {flops/us/1e6:7.1f} TFLOP/s (causal FLOPs)", flush=True)
