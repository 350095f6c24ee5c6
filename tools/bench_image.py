"""CLIP eval-transform throughput: CLIPImageProcessor on the GPU against torchvision + Pillow on the host.

Seeded synthetic RGB images in a fixed mix of decoded sizes (per 16 images: 5 x 500x375, 6 x 640x480, 4 x 1024x768 and
1 x 4000x3000, the last standing for full-resolution camera images).  Reports, for batches of 64 and 256:
  - kernel: GPU time of the two preprocessing kernels (torch.profiler), images already on the device;
  - h2d:    the one pinned host-to-device copy of the batch's pixels (CUDA events);
  - e2e:    host clock from decoded PIL images to the device vision_x, synchronised;
and the host transform in images/s on 1 thread and on os.cpu_count() worker processes, whether the timed GPU outputs
equal the host outputs bit for bit, and the card's name and power limit."""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from PIL import Image

MIX = [(375, 500)] * 5 + [(480, 640)] * 6 + [(768, 1024)] * 4 + [(3000, 4000)]
MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)


def images(n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        h, w = MIX[i % len(MIX)]
        # smooth content plus noise: resampling costs the same for any content
        base = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3), dtype=np.uint8).repeat(8, 0).repeat(8, 1)[:h, :w]
        out.append(Image.fromarray(base ^ rng.integers(0, 16, (1, w, 3), dtype=np.uint8), "RGB"))
    return out


def host_transform(S):
    from torchvision import transforms as T
    return T.Compose([T.Resize(S, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(S),
                      lambda im: im.convert("RGB"), T.ToTensor(), T.Normalize(MEAN, STD)])


_worker_imgs = None


def _init_worker(S):
    global _worker_imgs, _worker_tf
    torch.set_num_threads(1)
    _worker_imgs = images(len(MIX), seed=1)
    _worker_tf = host_transform(S)


def _work(i):
    _worker_tf(_worker_imgs[i % len(_worker_imgs)])
    return i


def host_rate(S, procs, n):
    if procs == 1:
        _init_worker(S)
        t0 = time.perf_counter()
        for i in range(n):
            _work(i)
        return n / (time.perf_counter() - t0)
    with mp.get_context("fork").Pool(procs, initializer=_init_worker, initargs=(S,)) as pool:
        pool.map(_work, range(procs * 2), chunksize=1)  # warm every worker
        t0 = time.perf_counter()
        pool.map(_work, range(n), chunksize=1)
        return n / (time.perf_counter() - t0)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--host-images", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_image needs a CUDA device")
    from open_flamingo_b200 import CLIPImageProcessor, ops
    S = args.size
    torch.cuda.set_device(0)
    proc = CLIPImageProcessor(S, MEAN, STD)
    res = {"card": card(), "image_size": S, "mix": "5x500x375 6x640x480 4x1024x768 1x4000x3000 per 16"}
    imgs_all = images(256)
    for n in (64, 256):
        imgs = imgs_all[:n]
        nbytes = sum(im.size[0] * im.size[1] * 3 for im in imgs)
        out = torch.empty(n, 3, S, S, device="cuda")
        # end to end: decoded PIL images -> device vision_x
        for _ in range(2):
            proc.batch(imgs, out=out)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.iters):
            proc.batch(imgs, out=out)
        torch.cuda.synchronize()
        e2e = (time.perf_counter() - t0) / args.iters
        # the one host-to-device copy
        pinned = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        dev = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dev.copy_(pinned, non_blocking=True)
        e0.record()
        for _ in range(args.iters):
            dev.copy_(pinned, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        h2d = e0.elapsed_time(e1) / args.iters / 1e3
        # the kernel pair on device-resident pixels
        dimgs = [torch.from_numpy(np.asarray(im)).cuda() for im in imgs]
        ops.clip_preprocess(dimgs, S, MEAN, STD, out=out)
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                ops.clip_preprocess(dimgs, S, MEAN, STD, out=out)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.events():
            if "image_resample" in ev.name and ev.device_type == torch.autograd.DeviceType.CUDA:
                key = "first" if "first" in ev.name else "second"
                kern[key] = kern.get(key, 0.0) + ev.time_range.elapsed_us() / 1e6 / args.iters
        kt = sum(kern.values())
        # bit-exactness of the timed output against the host transform
        tf = host_transform(S)
        want = torch.stack([tf(im) for im in imgs])
        exact = bool(torch.equal(out.cpu().view(torch.int32), want.view(torch.int32)))
        res[f"batch{n}"] = {
            "source_MB": round(nbytes / 1e6, 1),
            "kernel_ms": round(kt * 1e3, 3), "kernel_first_ms": round(kern.get("first", 0) * 1e3, 3),
            "kernel_second_ms": round(kern.get("second", 0) * 1e3, 3), "kernel_images_per_s": round(n / kt) if kt else None,
            "h2d_ms": round(h2d * 1e3, 3), "h2d_GB_per_s": round(nbytes / h2d / 1e9, 1),
            "e2e_ms": round(e2e * 1e3, 2), "e2e_images_per_s": round(n / e2e), "bit_exact_vs_host": exact}
        print(json.dumps({f"batch{n}": res[f"batch{n}"]}), flush=True)
    cpus = os.cpu_count()
    res["host_cpus"] = cpus
    res["host_1thread_images_per_s"] = round(host_rate(S, 1, args.host_images), 1)
    res["host_all_procs_images_per_s"] = round(host_rate(S, cpus, max(args.host_images, 4 * cpus)), 1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
