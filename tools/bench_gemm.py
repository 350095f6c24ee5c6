"""Per-shape GEMM timing and an L2 read-bandwidth probe (H100).

    python tools/bench_gemm.py [--shapes rows.json] [--top 10] [--launches 20] [--out result.json]

--shapes takes the table `bench.py --gemm-shapes` writes; without it the OF-3B training-step shapes below are timed.
Each distinct (layout, epilogue, M, N, K, splits) runs in isolation: `--launches` launches captured in one CUDA
graph, replayed, timed with CUDA events.  Per shape it reports TFLOP/s and the modelled L2 -> shared-memory operand
traffic, for the tile the library picks:
  128 x 128 tile           : (128 + 128) x 64 x 2 B per CTA k-block, 2.1 MFLOP
  128 x 256 on a 2-CTA pair: (128 + 128) x 64 x 2 B read from L2 per CTA k-block (B arrives by multicast), 4.2 MFLOP
The pick is modelled as the library makes it, with every SM pair as one cluster slot (the library asks the
occupancy API, which gives 66 on a 132-SM H100).

The L2 probe sums a 24 MB fp32 tensor, which stays resident in the 50 MB L2, in a replayed graph.  A torch
reduction is not a bandwidth-optimal reader, so its rate is a lower bound on what L2 can deliver.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from open_flamingo_b200 import _lib as L  # noqa: E402
from open_flamingo_b200 import ops  # noqa: E402

# OF-3B step (B = 32, T_txt = 256: 8192 LM tokens; 2048-wide MPT blocks, 4x FFN), forward and backward layouts:
# (epi, a_mn, b_mn, M, N, K, splits)
OF3B_SHAPES = [
    (L.EPI_GELU_DUAL, 0, 0, 8192, 8192, 2048, 1),      # FFN up, forward
    (L.EPI_GATE_RESID_F32, 0, 0, 8192, 2048, 8192, 1),  # FFN down + gated residual, forward
    (L.EPI_STORE_BF16, 0, 1, 8192, 8192, 2048, 1),     # dgrad of FFN down
    (L.EPI_DGELU_BF16, 0, 1, 8192, 8192, 2048, 1),     # dgrad of FFN down through GELU'
    (L.EPI_STORE_BF16, 0, 1, 8192, 2048, 8192, 1),     # dgrad of FFN up
    (L.EPI_STORE_F32, 1, 1, 2048, 8192, 8192, 1),      # wgrad of FFN down
    (L.EPI_STORE_F32, 1, 1, 8192, 2048, 8192, 1),      # wgrad of FFN up
    (L.EPI_STORE_BF16, 0, 0, 8192, 6144, 2048, 1),     # fused QKV projection
    (L.EPI_STORE_BF16, 0, 0, 8192, 2048, 2048, 1),     # attention out projection
    (L.EPI_ATOMIC_F32, 1, 1, 2048, 2048, 8192, 1),     # wgrad, atomic
]
PROBE_BYTES = 24 << 20


def pick_wide(m, n, k, splits, sms):
    total_kb = (k + 63) // 64
    per_split = -(-total_kb // max(1, min(splits, total_kb)))
    splits = -(-total_kb // per_split)
    shortest = total_kb - (splits - 1) * per_split
    return ((m + 127) // 128 + 1) // 2 * ((n + 255) // 256) * splits >= sms // 2 and shortest >= 4


def l2_bytes(m, n, k, splits, sms):
    kb = (k + 63) // 64
    if pick_wide(m, n, k, splits, sms):
        ctas = 2 * (((m + 127) // 128 + 1) // 2) * ((n + 255) // 256)
    else:
        ctas = ((m + 127) // 128) * ((n + 127) // 128)
    return ctas * kb * (128 + 128) * 64 * 2


def make_call(epi, a_mn, b_mn, m, n, k, splits, gen):
    dev = "cuda"
    a = torch.randn((k, m) if a_mn else (m, k), generator=gen, device=dev).to(torch.bfloat16)
    b = torch.randn((k, n) if b_mn else (n, k), generator=gen, device=dev).to(torch.bfloat16)
    kw = dict(a_mn=bool(a_mn), b_mn=bool(b_mn), epi=epi, splits=splits)
    f32_out = epi in (L.EPI_STORE_F32, L.EPI_ATOMIC_F32, L.EPI_GATE_RESID_F32, L.EPI_BIAS_RESID_F32)
    kw["out"] = torch.zeros((m, n), device=dev, dtype=torch.float32 if f32_out else torch.bfloat16)
    if epi in (L.EPI_BIAS_BF16, L.EPI_BIAS_QGELU_BF16, L.EPI_BIAS_RESID_F32, L.EPI_BIAS_GELU_BF16):
        kw["bias"] = torch.randn(n, generator=gen, device=dev)
    if epi in (L.EPI_GELU_DUAL, L.EPI_GATE_RESID_F32, L.EPI_BIAS_RESID_F32):
        kw["out2"] = torch.empty((m, n), device=dev, dtype=torch.bfloat16)
    if epi in (L.EPI_GATE_RESID_F32, L.EPI_BIAS_RESID_F32):
        kw["aux"] = torch.randn((m, n), generator=gen, device=dev)
    if epi == L.EPI_GATE_RESID_F32:
        kw["gate"] = torch.tensor([0.5], device=dev)
    if epi == L.EPI_DGELU_BF16:
        kw["aux"] = torch.randn((m, n), generator=gen, device=dev).to(torch.bfloat16)
    return lambda: ops.gemm(a, b, **kw)


def time_graph(fn, launches, replays):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (replays * launches)   # ms per launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=None, help="JSON rows written by bench.py --gemm-shapes")
    ap.add_argument("--top", type=int, default=10, help="with --shapes: the rows with the most ms per step")
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--replays", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm.py needs a GPU")
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    if args.shapes:
        rows = json.load(open(args.shapes))[:args.top]
        shapes = [(r["epi"], r["a_mn"], r["b_mn"], r["M"], r["N"], r["K"], r["splits"]) for r in rows]
    else:
        shapes = OF3B_SHAPES
    gen = torch.Generator(device="cuda").manual_seed(0)
    results = []
    for shape in shapes:
        epi, a_mn, b_mn, m, n, k, splits = shape
        ms = time_graph(make_call(*shape, gen), args.launches, args.replays)
        flop = 2.0 * m * n * k
        by = l2_bytes(m, n, k, splits, sms)
        r = {"epi": epi, "a_mn": a_mn, "b_mn": b_mn, "M": m, "N": n, "K": k, "splits": splits,
             "tile": "128x256x2" if pick_wide(m, n, k, splits, sms) else "128x128", "us": ms * 1e3,
             "TFLOP/s": flop / (ms * 1e-3) / 1e12, "model_L2_TB/s": by / (ms * 1e-3) / 1e12}
        results.append(r)
        print(json.dumps(r), flush=True)
    x = torch.randn(PROBE_BYTES // 4, device="cuda")
    out = torch.empty((), device="cuda")
    probe_ms = time_graph(lambda: torch.sum(x, 0, out=out), 50, 10)
    probe = {"l2_read_lower_bound_TB/s": PROBE_BYTES / (probe_ms * 1e-3) / 1e12, "bytes": PROBE_BYTES,
             "method": "torch.sum over a 24 MB fp32 tensor resident in L2, 50 launches per graph replay"}
    print(json.dumps(probe), flush=True)
    line = {"gpu": props.name, "sms": sms, "shapes": results, "l2_probe": probe}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
