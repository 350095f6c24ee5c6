"""GPU: OpenFlamingo-4B at its real dimensions -- ViT-L/14, a RedPajama-INCITE-3B-shaped GPT-NeoX LM (D 2560, 32 heads
of 80, 32 layers, FFN 10240), a gated block before every 2nd layer -- at 4 x (2 images, 256 tokens).

Parity: the same three evaluations and the same rule as test_fullsize_parity_gpu.py (ref = the oracle in fp32, amp =
the oracle under autocast(bf16), ours = the product under the same autocast): logits, loss, the gradient of every
trainable tensor and the hidden-state gradient at every decoder position satisfy err(ours, ref) <= 2 x err(amp, ref)
(+ 1e-3) with cosine >= 0.999, and the tanh gates are checked as a population.  The oracle runs HF's GPTNeoXLayer
through its pre-hooks, which take the hidden states positionally, as GPTNeoXModel passes them: no NeoX-specific keyword
is needed.  Ours runs every frozen block through lm_blocks.FrozenNeoXBlockFn; the test checks that HF's attention
never runs on the product side.

Reproducibility: one FlatTrainer step (forward, backward, clip, AdamW) run twice from the same parameters and optimizer
state ends with bit-identical loss, gradients and parameters.

The model (4 B parameters in fp32) and the oracle's fp32 copy of the frozen LM take about 32 GB together, so results
that are kept for comparison (three copies of ~1 B trainable gradients per batch) are moved to host memory as soon as
they are made, and every gradient is released once copied."""
import gc

import pytest
import torch

from test_fullsize_parity_gpu import VIT_L14, _batch, _compare, _oracle_of, _run_oracle, _run_ours

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _of4b(seed):
    from open_flamingo_b200.testing import NEOX_3B, build_flamingo
    model, _, tok = build_flamingo(VIT_L14, None, neox_kw=NEOX_3B, cross_attn_every_n_layers=2, device="cuda",
                                   gate_init=1.0, seed=seed)
    model.train()
    assert sum(layer is not None for layer in model.lang_encoder.gated_cross_attn_layers) == 16
    return model, tok


def _release_cached_memory():
    gc.collect()
    torch.cuda.empty_cache()


def _to_host(res):
    logits, loss, grads, hidden = res
    return (logits.cpu(), loss.cpu(), {k: g.cpu() for k, g in grads.items()},
            {k: h.cpu() for k, h in hidden.items()})


def test_of4b_4x_2img_256tok_against_the_oracle():
    from transformers.models.gpt_neox import modeling_gpt_neox as M
    from open_flamingo_b200.testing import NEOX_3B
    _release_cached_memory()
    model, tok = _of4b(0)
    orc, sd, trainable = _oracle_of(model, 2)
    calls = {"ours": 0}
    hf_forward = M.GPTNeoXAttention.forward

    def counted(self, *a, **k):
        calls["ours"] += 1
        return hf_forward(self, *a, **k)

    def runs():
        for seed in (6, 16):
            b = _batch(tok, 4, 2, 256, NEOX_3B["vocab_size"], seed=seed, first_image_at=5)
            M.GPTNeoXAttention.forward = counted
            try:
                ours = _to_host(_run_ours(model, b))
            finally:
                M.GPTNeoXAttention.forward = hf_forward
            model.zero_grad(set_to_none=True)
            amp_, ref = (_to_host(_run_oracle(orc, sd, trainable, b, amp=a)) for a in (True, False))
            for k in trainable:
                sd[k].grad = None
            yield ours, amp_, ref

    _compare("OF-4B 4x(2 img, 256 tok)", runs(), trainable)
    assert calls["ours"] == 0, f"HF's GPTNeoXAttention ran {calls['ours']} times on the product side"
    del model, orc, sd
    torch.cuda.empty_cache()


def test_of4b_flat_trainer_step_is_bitwise_reproducible():
    from open_flamingo_b200.testing import NEOX_3B
    from open_flamingo_b200.train import FlatTrainer
    _release_cached_memory()
    model, tok = _of4b(1)
    trainer = FlatTrainer(model, lr=1e-4, weight_decay=0.1, max_grad_norm=1.0)
    b = _batch(tok, 4, 2, 256, NEOX_3B["vocab_size"], seed=3)
    params0 = trainer.bucket.params.detach().cpu()

    def step():
        trainer.zero_grad()
        with torch.autocast("cuda", dtype=bf16):
            out = model(vision_x=b["vision_x"], lang_x=b["lang_x"], attention_mask=b["attention_mask"],
                        labels=b["labels"])
        out.loss.backward()
        trainer.step()
        torch.cuda.synchronize()
        return out.loss.detach().float().cpu(), trainer.bucket.grads.detach().cpu(), \
            trainer.bucket.params.detach().cpu()

    loss_a, grads_a, params_a = step()
    # back to the initial parameters and an empty optimizer state
    with torch.no_grad():
        trainer.bucket.params.copy_(params0.to(trainer.bucket.params.device))
        trainer.exp_avg.zero_()
        trainer.exp_avg_sq.zero_()
        trainer.step_dev.zero_()
    trainer.step_count = 0
    trainer.refresh_w16()
    loss_b, grads_b, params_b = step()
    assert torch.isfinite(grads_a).all() and grads_a.norm().item() > 0
    assert not torch.equal(params_a, params0), "the step changed no parameter"
    assert torch.equal(loss_a, loss_b), (loss_a.item(), loss_b.item())
    assert torch.equal(grads_a, grads_b), "gradients differ between two identical steps"
    assert torch.equal(params_a, params_b), "parameters differ between two identical steps"
