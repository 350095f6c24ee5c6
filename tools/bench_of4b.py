"""OpenFlamingo-4B (ViT-L/14 + RedPajama-INCITE-3B, a GPT-NeoX LM, cross-attention every 2nd layer) on the kernels.

  python tools/bench_of4b.py [--batch 4] [--t_txt 256] [--steps 6] [--gen-tokens 16] [--out DIR]

Measures, in one process on one GPU (random-init weights at the released dims; build_neox):
  train  tokens/s of the training step (autocast bf16 forward + backward + FlatTrainer.step), frozen LM blocks on the
         kernels (lm_blocks.FrozenNeoXBlockFn) vs lm_blocks.ENABLED = False (HF's GPTNeoXLayer in eager PyTorch),
         timed in alternating rounds so that both see the same clocks;
  decode ms per generated token of Flamingo.generate (greedy, B = 1, and 3 beams over B = 8) under autocast, in three
         alternating arms: kernels (KVCache, eager steps, ops.attn_decode at head_dim 80), graph
         (cache_implementation="static": one CUDA graph replay per token, decode_graph) and HF (DynamicCache, sdpa).
         For the graph arm also the GPU time of one replayed step between CUDA events, the capture time, and whether
         its tokens equal the kernels arm's.
Prints one JSON line with the card's name and power limit (nvidia-smi), as bench.py records them; --out writes it there
too.  The training batch is (batch, 2 images, t_txt tokens); if it does not fit, pass a smaller --batch.
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

VIT_L14 = dict(image_size=224, patch_size=14, width=1024, layers=24, heads=16, output_dim=768)


def gpu_identity():
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                            "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or None
    except Exception:
        return None


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--t_img", type=int, default=2)
    ap.add_argument("--t_txt", type=int, default=256)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gen-tokens", type=int, default=16)
    ap.add_argument("--layers", type=int, default=None, help="LM depth (default: the released 32)")
    ap.add_argument("--decode-only", action="store_true", help="skip the training measurement")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from open_flamingo_b200.testing import NEOX_3B, build_flamingo
    assert torch.cuda.is_available(), "bench_of4b measures on a GPU"
    torch.cuda.set_device(0)
    neox = dict(NEOX_3B)
    if args.layers:
        neox["num_hidden_layers"] = args.layers
    with contextlib.redirect_stdout(io.StringIO()):
        model, _, tok = build_flamingo(VIT_L14, None, neox_kw=neox, cross_attn_every_n_layers=2, device="cuda",
                                       gate_init=1.0, seed=0)
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    res = dict(model="of4b", gpu=gpu_identity(), lm_layers=neox["num_hidden_layers"], batch=args.batch,
               t_img=args.t_img, t_txt=args.t_txt)

    if not args.decode_only:
        train(args, model, media_id, eoc_id, neox, res)
    decode(args, model, media_id, res)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_of4b.json"), "w") as f:
            f.write(line + "\n")


def train(args, model, media_id, eoc_id, neox, res):
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.testing import synthetic_batch
    from open_flamingo_b200.train import FlatTrainer
    model.train()
    trainer = FlatTrainer(model, lr=1e-4, weight_decay=0.1, max_grad_norm=1.0)
    b = synthetic_batch(args.batch, args.t_img, args.t_txt, media_id, eoc_id, neox["vocab_size"],
                        image_size=VIT_L14["image_size"], seed=1)
    b = {k: v.cuda() for k, v in b.items()}

    def step():
        trainer.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(vision_x=b["vision_x"], lang_x=b["lang_x"], attention_mask=b["attention_mask"],
                        labels=b["labels"])
        out.loss.backward()
        trainer.step()

    times = {True: [], False: []}
    for on in (True, False):   # warm-up of both arms
        lm_blocks.ENABLED = on
        timed(step, 2)
    for _ in range(args.rounds):
        for on in (True, False):
            lm_blocks.ENABLED = on
            times[on].append(timed(step, args.steps))
    lm_blocks.ENABLED = True
    tok_step = args.batch * args.t_txt
    res["train_tok_s_kernels"] = round(tok_step / min(times[True]), 1)
    res["train_tok_s_hf_lm"] = round(tok_step / min(times[False]), 1)
    res["train_step_ms_kernels"] = [round(t * 1e3, 2) for t in times[True]]
    res["train_step_ms_hf_lm"] = [round(t * 1e3, 2) for t in times[False]]
    res["peak_mem_gb"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    del trainer
    torch.cuda.empty_cache()


def decode(args, model, media_id, res):
    from open_flamingo_b200 import lm_blocks
    model.eval()
    graphs = model.lang_encoder.decode_graphs
    capture_s = []
    capture = graphs._capture

    def timed_capture(*a, **k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        capture(*a, **k)
        torch.cuda.synchronize()
        capture_s.append(time.perf_counter() - t0)
    graphs._capture = timed_capture
    arms = {"kernels": (True, False), "graph": (True, True), "hf": (False, False)}   # (lm_blocks.ENABLED, static)
    g = torch.Generator().manual_seed(3)
    prompt = 32
    for name, B, beams in (("greedy_b1", 1, 1), ("beam3_b8", 8, 3)):
        vision_x = torch.randn(B, 1, 1, 3, 224, 224, generator=g).cuda()
        lang_x = torch.randint(0, 50000, (B, prompt), generator=g)
        lang_x[:, 0] = media_id
        lang_x = lang_x.cuda()

        def gen(arm, n):
            on, static = arms[arm]
            lm_blocks.ENABLED = on
            kw = dict(cache_implementation="static") if static else {}
            with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16):
                return model.generate(vision_x=vision_x, lang_x=lang_x, attention_mask=torch.ones_like(lang_x),
                                      max_new_tokens=n, min_new_tokens=n, num_beams=beams, use_cache=True,
                                      pad_token_id=0, eos_token_id=None, **kw)
        # every arm is warmed up at both lengths: the graph arm captures once per cache capacity (prompt + n rows,
        # bucketed), and both lengths below share one bucket
        n0 = len(capture_s)
        for arm in arms:
            timed(lambda: gen(arm, 2), 1)
            timed(lambda: gen(arm, args.gen_tokens + 1), 1)
        res[f"decode_graph_capture_ms_{name}"] = [round(t * 1e3, 1) for t in capture_s[n0:]]
        r0 = graphs.replays
        per = {arm: [] for arm in arms}
        for _ in range(args.rounds):
            for arm in arms:
                # per-token time: the difference of two lengths cancels the prompt and the vision encoder
                t_long, t_short = timed(lambda: gen(arm, args.gen_tokens + 1), 1), timed(lambda: gen(arm, 1), 1)
                per[arm].append((t_long - t_short) / args.gen_tokens)
        assert graphs.error is None and graphs.replays - r0 == args.rounds * args.gen_tokens, graphs.error
        for arm in arms:
            res[f"decode_ms_per_token_{name}_{arm}"] = round(min(per[arm]) * 1e3, 3)
        res[f"decode_graph_tokens_equal_kernels_{name}"] = bool(torch.equal(
            gen("kernels", args.gen_tokens), gen("graph", args.gen_tokens)))
        # GPU time of one replayed step: the last key's graph, replayed between events (it rewrites its last row)
        graph = next(reversed(graphs.entries.values())).graph
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        reps = 20
        graph.replay()
        ev[0].record()
        for _ in range(reps):
            graph.replay()
        ev[1].record()
        torch.cuda.synchronize()
        res[f"decode_graph_step_gpu_ms_{name}"] = round(ev[0].elapsed_time(ev[1]) / reps, 3)
        graphs.clear()
    lm_blocks.ENABLED = True
    graphs._capture = capture


if __name__ == "__main__":
    main()
