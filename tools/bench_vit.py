"""Vision-tower forward throughput: ViT-L/14 (head width 64, media attention core) against the LaION towers ViT-H/14,
ViT-g/14 and ViT-bigG/14 (head widths 80, 88, 104: ops.rope_pack + the head_dim-128 dense core on zero-padded heads).

  python tools/bench_vit.py [--n 64] [--steps 10] [--warmup 3] [--rounds 3] [--out DIR]

Random-init towers at the open_clip dims (factory._OPEN_CLIP_VISION_CFG), 224 px, N images per forward, as
Flamingo._encode_vision_x calls them (no_grad).  Reports per tower:
  - images/s of the forward, timed with CUDA events over `steps` forwards after `warmup`, best and median of `rounds`;
  - in a separate profiled pass (torch.profiler, CUDA activity) after all timing: the share of the tower's kernel time
    spent in the attention cores (attn_fwd_kernel, media or dense policy) and in the q/k/v packing (rope_pack_kernel);
and the card's name and power limit, read in the same run.  Prints one JSON line; --out also writes it there."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

TOWERS = ("ViT-L-14", "ViT-H-14", "ViT-g-14", "ViT-bigG-14")


def card():
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                        "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return r.stdout.strip() if r.returncode == 0 and r.stdout.strip() else "unknown"


def build(name):
    from open_flamingo_b200.src.factory import _OPEN_CLIP_VISION_CFG
    from open_flamingo_b200.src.vit import VisionTransformer
    torch.manual_seed(0)
    with torch.device("cuda"):
        return VisionTransformer(**_OPEN_CLIP_VISION_CFG[name], output_tokens=True).eval()


def time_forward(vit, x, steps, warmup, rounds):
    """Seconds per forward of each round, between CUDA events."""
    with torch.no_grad():
        for _ in range(warmup):
            vit(x)
        out = []
        for _ in range(rounds):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(steps):
                vit(x)
            t1.record()
            t1.synchronize()
            out.append(t0.elapsed_time(t1) / 1e3 / steps)
    return out


def kernel_shares(vit, x, iters):
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad():
        vit(x)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                vit(x)
            torch.cuda.synchronize()
    total = attn = pack = 0.0
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = ev.time_range.elapsed_us()
        total += us
        if "attn_fwd_kernel" in ev.name:
            attn += us
        elif "rope_pack_kernel" in ev.name:
            pack += us
    return dict(kernel_ms_per_forward=round(total / 1e3 / iters, 3), attention_share=round(attn / total, 4),
                pack_share=round(pack / total, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64, help="images per forward")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile-iters", type=int, default=3)
    ap.add_argument("--towers", default=",".join(TOWERS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vit measures on a GPU"
    torch.cuda.set_device(0)
    names = args.towers.split(",")
    x = torch.randn(args.n, 3, 224, 224, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    res = {}
    for name in names:
        vit = build(name)
        secs = sorted(time_forward(vit, x, args.steps, args.warmup, args.rounds))
        res[name] = dict(head_dim=vit.width // vit.heads, layers=len(vit.transformer.resblocks),
                         images_per_s_best=round(args.n / secs[0], 1),
                         images_per_s_median=round(args.n / secs[len(secs) // 2], 1),
                         ms_per_forward_best=round(secs[0] * 1e3, 2))
        del vit
        torch.cuda.empty_cache()
    for name in names:   # profiled after every timed round, so tracing never overlaps a timing
        vit = build(name)
        res[name].update(kernel_shares(vit, x, args.profile_iters))
        del vit
        torch.cuda.empty_cache()
    line = json.dumps(dict(bench="vit_forward", gpu=card(), n_images=args.n, image_size=224, steps=args.steps,
                           warmup=args.warmup, rounds=args.rounds, towers=res))
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_vit.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
