"""GPU: OpenFlamingo-9B v1 widths -- ViT-L/14 and a LLaMA-7B-shaped LM (D 4096, 32 heads of 128, FFN 11008, RMSNorm
eps 1e-6), a gated block before every 4th layer, at 2 x (3 images, 192 tokens) per batch.

Parity, on 8 of LLaMA-7B's 32 layers over four batches: the three evaluations and the rule of
test_fullsize_parity_gpu.py (ref = the oracle in fp32, amp = the oracle under autocast(bf16), ours = the product under
the same autocast): logits, loss, the gradient of every trainable tensor and the hidden-state gradient at every decoder
position satisfy err(ours, ref) <= 2 x err(amp, ref) (+ 1e-3) with cosine >= 0.999, and the tanh gates are checked as a
population.  The oracle runs HF's LlamaDecoderLayer through its pre-hooks; ours runs every frozen block through
lm_blocks.FrozenLlamaBlockFn, and HF's attention never runs on the product side.

Why 8 layers, four batches and unit-variance token embeddings:
  - With HF's 0.02 embedding init the residual stream entering the first blocks is about 60 times smaller than their
    branch outputs, and the first RMSNorms amplify bf16 rounding in the backward.  At 16 layers the hidden-state
    gradients of ours then reached only cosine 0.998 against the 0.999 floor (H100 80GB, 700 W).
  - The error of both bf16 arms grows with depth.  At 16 layers with unit embeddings a few trainable gradients of ours
    still fell to cosine 0.998-0.999.
  - The gate rules take a median and an rms over the gate population: 2 gates per gated block and batch.  With two
    batches at 8 layers that is 8 gates, and their median relative error (4.3e-2) exceeded 2 x autocast's (4.1e-2);
    four batches make it 16.

Reproducibility, on 16 layers: one FlatTrainer step run twice from the same parameters and optimizer state ends with
bit-identical loss, gradients and parameters.

Results kept for comparison are moved to host memory as soon as they are made."""
import gc

import pytest
import torch

from test_fullsize_parity_gpu import VIT_L14, _batch, _compare, _oracle_of, _run_oracle, _run_ours

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
EVERY = 4
PARITY_LAYERS, PARITY_SEEDS = 8, (6, 16, 26, 36)
REPRO_LAYERS = 16


def _of9b_v1_widths(seed, layers):
    from open_flamingo_b200.testing import LLAMA_7B, build_flamingo
    model, _, tok = build_flamingo(VIT_L14, None, llama_kw=dict(LLAMA_7B, num_hidden_layers=layers),
                                   cross_attn_every_n_layers=EVERY, device="cuda", gate_init=1.0, seed=seed)
    with torch.no_grad():   # unit-variance token embeddings (see the module docstring)
        emb = model.lang_encoder.get_input_embeddings().weight
        emb.normal_(generator=torch.Generator(device="cuda").manual_seed(seed))
    model.train()
    assert sum(layer is not None for layer in model.lang_encoder.gated_cross_attn_layers) == layers // EVERY
    return model, tok


def _to_host(res):
    logits, loss, grads, hidden = res
    return (logits.cpu(), loss.cpu(), {k: g.cpu() for k, g in grads.items()},
            {k: h.cpu() for k, h in hidden.items()})


def parity_runs(model, tok, orc, sd, trainable, calls):
    """(ours, amp, ref) per batch of PARITY_SEEDS, on the host; counts HF LlamaAttention calls on the product side."""
    from transformers.models.llama import modeling_llama as M
    from open_flamingo_b200.testing import LLAMA_7B
    hf_forward = M.LlamaAttention.forward

    def counted(self, *a, **k):
        calls["ours"] += 1
        return hf_forward(self, *a, **k)

    for seed in PARITY_SEEDS:
        b = _batch(tok, 2, 3, 192, LLAMA_7B["vocab_size"], seed=seed, first_image_at=5)
        M.LlamaAttention.forward = counted
        try:
            ours = _to_host(_run_ours(model, b))
        finally:
            M.LlamaAttention.forward = hf_forward
        model.zero_grad(set_to_none=True)
        amp_, ref = (_to_host(_run_oracle(orc, sd, trainable, b, amp=a)) for a in (True, False))
        for k in trainable:
            sd[k].grad = None
        yield ours, amp_, ref


def test_of9b_v1_widths_4x_2x_3img_192tok_against_the_oracle():
    gc.collect()
    torch.cuda.empty_cache()
    model, tok = _of9b_v1_widths(0, PARITY_LAYERS)
    orc, sd, trainable = _oracle_of(model, EVERY)
    calls = {"ours": 0}
    _compare(f"OF-9B v1 widths, {PARITY_LAYERS} layers, 4 batches of 2x(3 img, 192 tok)",
             parity_runs(model, tok, orc, sd, trainable, calls), trainable)
    assert calls["ours"] == 0, f"HF's LlamaAttention ran {calls['ours']} times on the product side"
    del model, orc, sd
    torch.cuda.empty_cache()


def test_of9b_v1_flat_trainer_step_is_bitwise_reproducible():
    from transformers.models.llama import modeling_llama as M
    from open_flamingo_b200.testing import LLAMA_7B
    from open_flamingo_b200.train import FlatTrainer
    gc.collect()
    torch.cuda.empty_cache()
    model, tok = _of9b_v1_widths(1, REPRO_LAYERS)
    trainer = FlatTrainer(model, lr=1e-4, weight_decay=0.1, max_grad_norm=1.0)
    b = _batch(tok, 2, 3, 192, LLAMA_7B["vocab_size"], seed=3)
    params0 = trainer.bucket.params.detach().cpu()
    calls = {"hf_attn": 0}
    hf_forward = M.LlamaAttention.forward

    def counted(self, *a, **k):
        calls["hf_attn"] += 1
        return hf_forward(self, *a, **k)

    def step():
        trainer.zero_grad()
        M.LlamaAttention.forward = counted
        try:
            with torch.autocast("cuda", dtype=bf16):
                out = model(vision_x=b["vision_x"], lang_x=b["lang_x"], attention_mask=b["attention_mask"],
                            labels=b["labels"])
        finally:
            M.LlamaAttention.forward = hf_forward
        out.loss.backward()
        trainer.step()
        torch.cuda.synchronize()
        return out.loss.detach().float().cpu(), trainer.bucket.grads.detach().cpu(), \
            trainer.bucket.params.detach().cpu()

    loss_a, grads_a, params_a = step()
    with torch.no_grad():   # back to the initial parameters and an empty optimizer state
        trainer.bucket.params.copy_(params0.to(trainer.bucket.params.device))
        trainer.exp_avg.zero_()
        trainer.exp_avg_sq.zero_()
        trainer.step_dev.zero_()
    trainer.step_count = 0
    trainer.refresh_w16()
    loss_b, grads_b, params_b = step()
    assert calls["hf_attn"] == 0, f"HF's LlamaAttention ran {calls['hf_attn']} times on the product side"
    assert torch.isfinite(grads_a).all() and grads_a.norm().item() > 0
    assert not torch.equal(params_a, params0), "the step changed no parameter"
    assert torch.equal(loss_a, loss_b), (loss_a.item(), loss_b.item())
    assert torch.equal(grads_a, grads_b), "gradients differ between two identical steps"
    assert torch.equal(params_a, params_b), "parameters differ between two identical steps"
