"""OpenFlamingo-9B v1 (ViT-L/14 + LLaMA-7B, cross-attention every 4th layer) on the kernels.

  python tools/bench_llama.py [--batch 2] [--t_img 3] [--t_txt 192] [--steps 3] [--gen-tokens 16] [--out DIR]

Measures, in one process on one GPU (random-init weights at the released dims; build_llama):
  train  tokens/s of the training step (autocast bf16 forward + backward + FlatTrainer.step), frozen LM blocks on the
         kernels (lm_blocks.FrozenLlamaBlockFn) vs lm_blocks.ENABLED = False (HF's LlamaDecoderLayer in eager PyTorch),
         timed in alternating rounds so that both see the same clocks; peak memory (bench_of4b's train());
  decode ms per generated token of Flamingo.generate (greedy, B = 1, and 3 beams over B = 8) under autocast, in two
         alternating arms: kernels (KVCache, eager steps, ops.attn_decode at head_dim 128) and HF (DynamicCache, sdpa),
         and whether the two arms chose the same tokens.
Prints one JSON line with the card's name, power limit and maximum SM clock (nvidia-smi); --out writes it there too.
"""
import argparse
import contextlib
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.bench_of4b import VIT_L14, gpu_identity, timed, train  # noqa: E402

EVERY = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--t_img", type=int, default=3)
    ap.add_argument("--t_txt", type=int, default=192)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gen-tokens", type=int, default=16)
    ap.add_argument("--layers", type=int, default=None, help="LM depth (default: LLaMA-7B's 32)")
    ap.add_argument("--decode-only", action="store_true", help="skip the training measurement")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from open_flamingo_b200.testing import LLAMA_7B, build_flamingo
    assert torch.cuda.is_available(), "bench_llama measures on a GPU"
    torch.cuda.set_device(0)
    llama = dict(LLAMA_7B)
    if args.layers:
        llama["num_hidden_layers"] = args.layers
    with contextlib.redirect_stdout(io.StringIO()):
        model, _, tok = build_flamingo(VIT_L14, None, llama_kw=llama, cross_attn_every_n_layers=EVERY, device="cuda",
                                       gate_init=1.0, seed=0)
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    res = dict(model="of9b-v1-llama7b", gpu=gpu_identity(), lm_layers=llama["num_hidden_layers"], batch=args.batch,
               t_img=args.t_img, t_txt=args.t_txt)
    if not args.decode_only:
        train(args, model, media_id, eoc_id, llama, res)
    decode(args, model, media_id, llama, res)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_llama.json"), "w") as f:
            f.write(line + "\n")


def decode(args, model, media_id, llama, res):
    from open_flamingo_b200 import lm_blocks
    model.eval()
    g = torch.Generator().manual_seed(3)
    prompt = 32
    for name, B, beams in (("greedy_b1", 1, 1), ("beam3_b8", 8, 3)):
        vision_x = torch.randn(B, 1, 1, 3, 224, 224, generator=g).cuda()
        lang_x = torch.randint(0, llama["vocab_size"], (B, prompt), generator=g)
        lang_x[:, 0] = media_id
        lang_x = lang_x.cuda()

        def gen(on, n):
            lm_blocks.ENABLED = on
            with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16):
                return model.generate(vision_x=vision_x, lang_x=lang_x, attention_mask=torch.ones_like(lang_x),
                                      max_new_tokens=n, min_new_tokens=n, num_beams=beams, use_cache=True,
                                      pad_token_id=0, eos_token_id=None)
        for on in (True, False):
            timed(lambda: gen(on, 2), 1)
            timed(lambda: gen(on, args.gen_tokens + 1), 1)
        per = {True: [], False: []}
        for _ in range(args.rounds):
            for on in (True, False):
                # per-token time: the difference of two lengths cancels the prompt and the vision encoder
                t_long, t_short = timed(lambda: gen(on, args.gen_tokens + 1), 1), timed(lambda: gen(on, 1), 1)
                per[on].append((t_long - t_short) / args.gen_tokens)
        res[f"decode_ms_per_token_{name}_kernels"] = round(min(per[True]) * 1e3, 3)
        res[f"decode_ms_per_token_{name}_hf"] = round(min(per[False]) * 1e3, 3)
        res[f"decode_tokens_equal_{name}"] = bool(torch.equal(gen(True, args.gen_tokens), gen(False, args.gen_tokens)))
    torch.cuda.reset_peak_memory_stats()
    gen(True, args.gen_tokens)
    res["peak_mem_gb_decode_beam3_b8_kernels"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    lm_blocks.ENABLED = True


if __name__ == "__main__":
    main()
