"""Decode-step benchmark: Flamingo.generate with the KV cache on the kernels versus HF's blocks and DynamicCache.

Workload: OF-3B dims (ViT-L/14 + MPT-1B, cross-attention every layer), random init, under autocast(bf16) and
inference_mode as in the reference's captioning / VQA evaluation.  Prompts carry 4 images and ~200 tokens, left-padded,
20 new tokens, at (B=1, greedy) and (B=8, num_beams=3).  The three arms ("kernels": lm_blocks.ENABLED with the growing
KVCache, "graph": the same with cache_implementation="static", one CUDA graph replay per token, "hf": the frozen blocks
on HF's own forward and DynamicCache) alternate within one run.

Reported per arm: prefill ms, ms per generated token, the share of a decode step spent in libofk GEMMs (CUDA event pairs
around every GEMM, in a separate pass; not measurable inside a graph), host time per decode step, and whether the
arms' tokens agree.  For the graph arm also: the capture time, and the first call (which captures) against later
calls.  Then the decode attention kernels alone (CUDA events over many launches): bytes moved (q + K/V rows + o) over
time, against the H100 SXM data-sheet 3.35 TB/s, for ofk_attn_decode and ofk_attn_decode_dev.  The card's name, power
limit and max SM clock are printed in the same run.

    python tools/bench_decode.py [--reps 3] [--new-tokens 20]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VIT_L14 = dict(image_size=224, patch_size=14, width=1024, layers=24, heads=16, output_dim=768)
HBM_BYTES_PER_S = 3.35e12


def gpu_identity():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if out else {"name": torch.cuda.get_device_name()}


@contextlib.contextmanager
def fast_lm(on):
    from open_flamingo_b200 import lm_blocks
    prev = lm_blocks.ENABLED
    lm_blocks.ENABLED = on
    try:
        yield
    finally:
        lm_blocks.ENABLED = prev


def prompts(B, tok, vocab, T=200, n_img=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    media = tok.encode("<image>")[-1]
    ids = torch.randint(0, vocab, (B, T), generator=g)
    att = torch.ones_like(ids)
    for b in range(B):
        pad = int(torch.randint(0, 40, (1,), generator=g)) if B > 1 else 0
        att[b, :pad] = 0
        ids[b, :pad] = 0
        span = T - pad
        for k in range(n_img):
            ids[b, pad + k * span // n_img] = media
    vision_x = torch.randn(B, n_img, 1, 3, 224, 224, generator=g)
    return vision_x.cuda(), ids.cuda(), att.cuda()


def generate(model, vision_x, ids, att, beams, new_tokens, static=False):
    kw = dict(cache_implementation="static") if static else {}
    with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16):
        return model.generate(vision_x=vision_x, lang_x=ids, attention_mask=att, max_new_tokens=new_tokens,
                              num_beams=beams, do_sample=False, use_cache=True, pad_token_id=0, eos_token_id=None,
                              min_new_tokens=new_tokens, **kw)


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t) * 1e3


class GemmEvents:
    """CUDA event pairs around every libofk GEMM call."""

    def __init__(self):
        self.pairs = []

    def __enter__(self):
        from open_flamingo_b200 import ops
        self.saved = (ops.gemm, ops.gemm_grouped)

        def wrap(fn):
            def w(*a, **k):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                r = fn(*a, **k)
                e1.record()
                self.pairs.append((e0, e1))
                return r
            return w
        ops.gemm, ops.gemm_grouped = wrap(ops.gemm), wrap(ops.gemm_grouped)
        return self

    def __exit__(self, *exc):
        from open_flamingo_b200 import ops
        ops.gemm, ops.gemm_grouped = self.saved

    def ms(self):
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in self.pairs)


def decode_steps(model, vision_x, ids, att, beams, steps, kernels, graph=False):
    """Manual decode loop (prefill, then `steps` single-token forwards with the cache): per-step GPU ms, host enqueue
    ms, and GEMM ms per step from event pairs in a second identical pass (None for the graph arm)."""
    from transformers import DynamicCache
    if beams > 1:
        vision_x, ids, att = (t.repeat_interleave(beams, 0) for t in (vision_x, ids, att))
    lm = model.lang_encoder

    def run(events=None):
        with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16), fast_lm(kernels):
            model.cache_media(input_ids=ids, vision_x=vision_x)
            cache = lm.make_kv_cache(capacity=ids.shape[1] + steps + 1 if graph else None) if kernels else \
                DynamicCache()
            assert kernels == (cache is not None and type(cache).__name__ == "KVCache")
            out = model(vision_x=None, lang_x=ids, attention_mask=att, clear_conditioned_layers=False,
                        past_key_values=cache, use_cache=True)
            nxt = out.logits[:, -1:].argmax(-1)
            a = att
            host, gpu = [], []
            ctx = events if events is not None else contextlib.nullcontext()
            torch.cuda.synchronize()
            with ctx:
                for _ in range(steps):
                    a = torch.cat([a, torch.ones_like(a[:, :1])], 1)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    t = time.perf_counter()
                    out = model(vision_x=None, lang_x=nxt, attention_mask=a, clear_conditioned_layers=False,
                                past_key_values=cache, use_cache=True)
                    host.append((time.perf_counter() - t) * 1e3)
                    e1.record()
                    gpu.append((e0, e1))
                    nxt = out.logits[:, -1:].argmax(-1)
            torch.cuda.synchronize()
            model.uncache_media()
            return sum(x.elapsed_time(y) for x, y in gpu) / steps, sum(host) / steps

    run()   # warm-up
    step_ms, host_ms = run()
    if graph:
        return step_ms, host_ms, None
    ev = GemmEvents()
    gemm_step_ms, _ = run(ev)
    return step_ms, host_ms, ev.ms() / steps / gemm_step_ms


def _graph_us(fn, reps):
    """Mean µs of `fn` over `reps` launches captured in one CUDA graph (the kernels' time, not the wrapper's)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            fn()
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def bench_kernel(reps=200):
    from open_flamingo_b200 import ops
    rows = []
    hd = 128
    for BH in (16, 384):
        H = 16
        B = BH // H
        D = H * hd
        for nk in (128, 512, 2048):
            buf = torch.randn(B, nk + 64, 2 * D, device="cuda").to(torch.bfloat16)
            q = torch.randn(B, D, device="cuda").to(torch.bfloat16)
            k, v = buf[:, :nk, :D], buf[:, :nk, D:]
            slopes = torch.rand(H, device="cuda")
            mask = torch.zeros(B, -(-nk // 8) * 8, dtype=torch.uint8, device="cuda")
            out = torch.empty(B, D, device="cuda", dtype=torch.bfloat16)
            nk_dev = torch.tensor([nk], device="cuda", dtype=torch.int32)
            ws = ops.decode_workspace(torch.device("cuda"), B, H, hd, nk)
            us = _graph_us(lambda: ops.attn_decode(q, k, v, H, hd, hd ** -0.5, key_mask=mask, slopes=slopes, out=out),
                           reps)
            us_dev = _graph_us(lambda: ops.attn_decode_dev(q, k, v, H, hd, hd ** -0.5, nk_dev, key_mask=mask,
                                                           slopes=slopes, out=out, workspace=ws), reps)
            nbytes = BH * hd * 2 * (2 + 2 * nk)   # q + K/V rows + o (the mask and slopes are < 1 %)
            rows.append(dict(BH=BH, nk=nk, head_dim=hd, us=round(us, 2), GBps=round(nbytes / us / 1e3, 1),
                             share_of_3_35TBps=round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3),
                             us_dev=round(us_dev, 2),
                             share_of_3_35TBps_dev=round(nbytes / (us_dev * 1e-6) / HBM_BYTES_PER_S, 3)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--new-tokens", type=int, default=20)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    import __graft_entry__  # noqa: F401
    from open_flamingo_b200.testing import MPT_1B, build_flamingo
    print(json.dumps({"gpu": gpu_identity()}), flush=True)
    print(json.dumps({"decode_kernel": bench_kernel()}), flush=True)

    model, _, tok = build_flamingo(VIT_L14, dict(MPT_1B), cross_attn_every_n_layers=1, device="cuda", gate_init=1.0,
                                   seed=0)
    model.eval().requires_grad_(False)
    vocab = MPT_1B["vocab_size"]
    arms = ("kernels", "graph", "hf")
    graphs = model.lang_encoder.decode_graphs
    capture_ms = []
    capture = graphs._capture

    def timed_capture(*a):
        torch.cuda.synchronize()
        t = time.perf_counter()
        capture(*a)
        torch.cuda.synchronize()
        capture_ms.append((time.perf_counter() - t) * 1e3)
    graphs._capture = timed_capture
    for B, beams in ((1, 1), (8, 3)):
        vision_x, ids, att = prompts(B, tok, vocab)
        res = {arm: {} for arm in arms}
        seqs = {}
        for arm in arms:      # warm-up every arm; the graph arm's first call captures
            with fast_lm(arm != "hf"):
                _, ms = timed(lambda: generate(model, vision_x, ids, att, beams, args.new_tokens, arm == "graph"))
            if arm == "graph":
                res[arm]["first_call_ms"] = round(ms, 2)
                res[arm]["capture_ms"] = round(capture_ms[-1], 2) if capture_ms else None
        for _ in range(args.reps):
            for arm in arms:
                with fast_lm(arm != "hf"):
                    _, t1 = timed(lambda: generate(model, vision_x, ids, att, beams, 1))
                    seqs[arm], tn = timed(lambda: generate(model, vision_x, ids, att, beams, args.new_tokens,
                                                           arm == "graph"))
                res[arm].setdefault("prefill_ms", []).append(t1)
                res[arm].setdefault("call_ms", []).append(tn)
                res[arm].setdefault("ms_per_token", []).append((tn - t1) / (args.new_tokens - 1))
        for arm in arms:
            step_ms, host_ms, gemm_share = decode_steps(model, vision_x, ids, att, beams, 16, arm != "hf",
                                                        arm == "graph")
            r = res[arm]
            r["prefill_ms"] = round(min(r["prefill_ms"]), 2)
            r["later_call_ms"] = round(min(r.pop("call_ms")), 2)
            r["ms_per_token"] = round(min(r["ms_per_token"]), 3)
            r["decode_step_gpu_ms"] = round(step_ms, 3)
            r["host_ms_per_step"] = round(host_ms, 3)
            r["gemm_share_of_step"] = None if gemm_share is None else round(gemm_share, 3)
        res["graph"]["replays"] = graphs.replays
        res["graph"]["captures"] = graphs.captures
        res["graph"]["error"] = None if graphs.error is None else repr(graphs.error)
        res["tokens_agree"] = bool(torch.equal(seqs["kernels"], seqs["hf"]))
        res["graph_tokens_equal_kernels"] = bool(torch.equal(seqs["graph"], seqs["kernels"]))
        print(json.dumps({"B": B, "num_beams": beams, "prompt_tokens": ids.shape[1], "images": 4,
                          "new_tokens": args.new_tokens, **res}), flush=True)


if __name__ == "__main__":
    main()
