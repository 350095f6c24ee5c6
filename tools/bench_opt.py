"""Flamingo with an OPT LM (ViT-L/14 + OPT-1.3B or OPT-2.7B, cross-attention every 4th layer) on the kernels.

  python tools/bench_opt.py [--lm opt-2.7b] [--batch 2] [--t_img 3] [--t_txt 192] [--steps 3] [--gen-tokens 16]
                            [--out DIR]

Measures, in one process on one GPU (random-init weights at the released dims; build_opt):
  train  tokens/s of the training step (autocast bf16 forward + backward + FlatTrainer.step) in train mode with the
         configs' residual dropout 0.1, frozen LM blocks on the kernels (lm_blocks.FrozenOptBlockFn, with
         ofk_dropout_resid_fwd / _bwd) vs lm_blocks.ENABLED = False (HF's OPTDecoderLayer in eager PyTorch), timed in
         alternating rounds so that both see the same clocks; peak memory (bench_of4b's train());
  decode ms per generated token of Flamingo.generate (greedy, B = 1, and 3 beams over B = 8) under autocast, kernels
         (KVCache, eager steps) against HF (DynamicCache, sdpa), and whether the two arms chose the same tokens
         (bench_llama's decode()).
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

from tools.bench_llama import decode  # noqa: E402
from tools.bench_of4b import VIT_L14, gpu_identity, train  # noqa: E402

EVERY = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lm", choices=("opt-1.3b", "opt-2.7b"), default="opt-2.7b")
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--t_img", type=int, default=3)
    ap.add_argument("--t_txt", type=int, default=192)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--gen-tokens", type=int, default=16)
    ap.add_argument("--layers", type=int, default=None, help="LM depth (default: the config's)")
    ap.add_argument("--decode-only", action="store_true", help="skip the training measurement")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from open_flamingo_b200.testing import OPT_1_3B, OPT_2_7B, build_flamingo
    assert torch.cuda.is_available(), "bench_opt measures on a GPU"
    torch.cuda.set_device(0)
    opt = dict(OPT_1_3B if args.lm == "opt-1.3b" else OPT_2_7B)
    if args.layers:
        opt["num_hidden_layers"] = args.layers
    with contextlib.redirect_stdout(io.StringIO()):
        model, _, tok = build_flamingo(VIT_L14, None, opt_kw=opt, cross_attn_every_n_layers=EVERY, device="cuda",
                                       gate_init=1.0, seed=0)
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    res = dict(model=f"flamingo-{args.lm}", gpu=gpu_identity(), lm_layers=opt["num_hidden_layers"],
               dropout=opt["dropout"], batch=args.batch, t_img=args.t_img, t_txt=args.t_txt)
    if not args.decode_only:
        train(args, model, media_id, eoc_id, opt, res)
    decode(args, model, media_id, opt, res)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_opt.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
