"""BASELINE configs[4]: PerceiverResampler isolation bench -- 64 latents x 4096 visual tokens x d=1024, 6 layers,
fwd+bwd on one GPU (U = 64 images), CUDA-event timed; prints achieved TFLOP/s against SURVEY section 8d's
algorithmic count (62.8 GFLOP/image forward; backward = 2x forward minus the media-row dgrad... which IS needed
for norm_media's affine gradients, so 3x forward is used)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from open_flamingo_b200 import _lib
from open_flamingo_b200.src.helpers import PerceiverResampler

U, v, D, n, depth = 64, int(os.environ.get("V", 4096)), 1024, 64, 6
torch.manual_seed(0)
m = PerceiverResampler(dim=D, depth=depth).cuda()
x = torch.randn(8, 8, 1, v, D, device="cuda").to(getattr(torch, os.environ.get("XDTYPE", "float32")))
w = torch.randn(8, 8, n, D, device="cuda")


def step():
    for p in m.parameters():
        p.grad = None
    y = m(x)
    (y * w).sum().backward()


for _ in range(int(os.environ.get("WARM", 3))):
    step()
torch.cuda.synchronize()
l0 = _lib.launch_count()
step()
launches = _lib.launch_count() - l0
# the 190 launches of a forward + backward are captured once and replayed (as bench.py does for the training step): an
# eager pass on a busy host is bound by the Python / ctypes time per launch, not by the kernels
graph = None
if os.environ.get("GRAPH", "1") == "1":
    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            step()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        graph.replay()
        torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        print(f"[bench_perceiver] CUDA-graph capture unavailable ({e!r}); timing eagerly", file=sys.stderr)
        graph = None
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
iters = int(os.environ.get("ITERS", 5))
e0.record()
for _ in range(iters):
    if graph is not None:
        graph.replay()
    else:
        step()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / iters
I = 512
fwd_per_image = depth * (2 * n * D * I + 2 * (v + n) * D * 2 * I + 4 * 8 * n * (v + n) * 64 + 2 * n * I * D + 16 * n * D * D)
flops = 3 * fwd_per_image * U
peak = 989.0   # TFLOP/s: NVIDIA data-sheet dense BF16 of the H100 SXM at 700 W (a peak, not a measured rate)
print(json.dumps({"workload": "PerceiverResampler isolation C5", "images": U, "visual_tokens": v, "dim": D, "latents": n,
                  "depth": depth, "ms_fwd_bwd": ms, "algorithmic_TFLOP": flops / 1e12, "achieved_TFLOPs": flops / ms / 1e9,
                  "peak_TFLOPs": peak, "frac": flops / ms / 1e9 / peak, "launches_per_step": launches, "cuda_graph": graph is not None}))
