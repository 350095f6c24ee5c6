"""GPU: OPT-1.3B widths (D 2048, 32 heads of 64, FFN 8192) and OPT-2.7B widths (D 2560, 32 heads of 80, FFN 10240)
with ViT-L/14, a gated block before every 4th layer, at 2 x (3 images, 192 tokens) per batch.

Parity, in eval-mode dropout (the LM's dropout set to 0, since the fp32 oracle would draw other masks), on 8 layers over
four batches: the three evaluations and the rule of test_fullsize_parity_gpu.py (ref = the oracle in fp32, amp = the
oracle under autocast(bf16), ours = the product under the same autocast): logits, loss, the gradient of every trainable
tensor and the hidden-state gradient at every decoder position satisfy err(ours, ref) <= 2 x err(amp, ref) (+ 1e-3)
with cosine >= 0.999, and the tanh gates are checked as a population.  HF's OPTAttention never runs on the product side.

Depth, batches and embeddings follow test_llama_fullsize_gpu.py, for its reasons: the error of both bf16 arms grows
with depth, so 8 layers keep the cosine floor meaningful; the gate rules take a median and an rms over the gate
population (2 gates per gated block and batch), and four batches at 8 layers make 16 gates; unit-variance token
embeddings keep the residual stream entering the first blocks from being dwarfed by their branch outputs, which would
let the first LayerNorms amplify bf16 rounding in the backward.

Reproducibility, with dropout 0.1 in train mode on 8 OPT-1.3B-wide layers: one FlatTrainer step run twice from the same
torch seed, parameters and optimizer state ends with bit-identical loss, gradients and parameters, and a
train.GraphedTrainStep replay from the same state and dropout (seed, offset) equals the eager step bit for bit.

Results kept for comparison are moved to host memory as soon as they are made."""
import gc

import pytest
import torch

from test_fullsize_parity_gpu import VIT_L14, _batch, _compare, _oracle_of
from test_llama_fullsize_gpu import _to_host

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
EVERY = 4
PARITY_LAYERS, PARITY_SEEDS = 8, (6, 16, 26, 36)
REPRO_LAYERS = 8


def _opt_widths(kw, seed, layers, dropout):
    from open_flamingo_b200.testing import build_flamingo
    model, _, tok = build_flamingo(VIT_L14, None, opt_kw=dict(kw, num_hidden_layers=layers, dropout=dropout),
                                   cross_attn_every_n_layers=EVERY, device="cuda", gate_init=1.0, seed=seed)
    with torch.no_grad():   # unit-variance token embeddings (see the module docstring)
        emb = model.lang_encoder.get_input_embeddings().weight
        emb.normal_(generator=torch.Generator(device="cuda").manual_seed(seed))
    model.train()
    assert sum(layer is not None for layer in model.lang_encoder.gated_cross_attn_layers) == layers // EVERY
    return model, tok


def _parity_runs(model, tok, orc, sd, trainable, calls, vocab):
    from transformers.models.opt import modeling_opt as M
    from test_fullsize_parity_gpu import _run_oracle, _run_ours
    hf_forward = M.OPTAttention.forward

    def counted(self, *a, **k):
        calls["ours"] += 1
        return hf_forward(self, *a, **k)

    for seed in PARITY_SEEDS:
        b = _batch(tok, 2, 3, 192, vocab, seed=seed, first_image_at=5)
        M.OPTAttention.forward = counted
        try:
            ours = _to_host(_run_ours(model, b))
        finally:
            M.OPTAttention.forward = hf_forward
        model.zero_grad(set_to_none=True)
        amp_, ref = (_to_host(_run_oracle(orc, sd, trainable, b, amp=a)) for a in (True, False))
        for k in trainable:
            sd[k].grad = None
        yield ours, amp_, ref


@pytest.mark.parametrize("which", ["OPT_1_3B", "OPT_2_7B"])
def test_opt_widths_4x_2x_3img_192tok_against_the_oracle(which):
    from open_flamingo_b200 import testing
    kw = getattr(testing, which)
    gc.collect()
    torch.cuda.empty_cache()
    model, tok = _opt_widths(kw, 0, PARITY_LAYERS, dropout=0.0)
    orc, sd, trainable = _oracle_of(model, EVERY)
    calls = {"ours": 0}
    _compare(f"{which} widths, {PARITY_LAYERS} layers, 4 batches of 2x(3 img, 192 tok)",
             _parity_runs(model, tok, orc, sd, trainable, calls, kw["vocab_size"]), trainable)
    assert calls["ours"] == 0, f"HF's OPTAttention ran {calls['ours']} times on the product side"
    del model, orc, sd
    torch.cuda.empty_cache()


def test_opt_dropout_training_step_is_reproducible_and_graph_replay_equals_eager():
    from open_flamingo_b200 import lm_blocks
    from open_flamingo_b200.testing import OPT_1_3B
    from open_flamingo_b200.train import FlatTrainer, GraphedTrainStep
    gc.collect()
    torch.cuda.empty_cache()
    model, tok = _opt_widths(OPT_1_3B, 1, REPRO_LAYERS, dropout=0.1)
    trainer = FlatTrainer(model, lr=1e-4, weight_decay=0.1, max_grad_norm=1.0)
    b = _batch(tok, 2, 3, 192, OPT_1_3B["vocab_size"], seed=3)
    params0 = trainer.bucket.params.detach().clone()

    def reset():
        with torch.no_grad():   # back to the initial parameters and an empty optimizer state
            trainer.bucket.params.copy_(params0)
            trainer.exp_avg.zero_()
            trainer.exp_avg_sq.zero_()
            trainer.step_dev.zero_()
        trainer.step_count = 0
        trainer.refresh_w16()

    def eager_step():
        trainer.zero_grad()
        with torch.autocast("cuda", dtype=bf16):
            out = model(vision_x=b["vision_x"], lang_x=b["lang_x"], attention_mask=b["attention_mask"],
                        labels=b["labels"])
        out.loss.backward()
        trainer.step()
        return out.loss.detach()

    def result(loss):
        torch.cuda.synchronize()
        return loss.float().cpu(), trainer.bucket.grads.detach().cpu(), trainer.bucket.params.detach().cpu()

    torch.manual_seed(5)
    a = result(eager_step())
    reset()
    torch.manual_seed(5)
    b_ = result(eager_step())
    assert torch.isfinite(a[1]).all() and a[1].norm().item() > 0
    assert not torch.equal(a[2], params0.cpu()), "the step changed no parameter"
    for x, y, what in zip(a, b_, ("loss", "gradients", "parameters")):
        assert torch.equal(x, y), f"{what} differ between two identical dropout steps"
    # another seed draws other masks
    reset()
    torch.manual_seed(6)
    c = result(eager_step())
    assert not torch.equal(a[1], c[1])

    reset()
    rng = lm_blocks.dropout_rng("cuda")
    step = GraphedTrainStep(model, trainer, b, warmup=1)
    assert step.ok, step.error
    start = torch.tensor([1234567, 40], dtype=torch.int64, device="cuda")
    reset()
    rng.state.copy_(start)
    g = result(step(b))
    reset()
    rng.state.copy_(start)
    e = result(eager_step())
    for x, y, what in zip(g, e, ("loss", "gradients", "parameters")):
        assert torch.equal(x, y), f"{what}: graph replay differs from the eager step"
    step.graph = None
    del model, trainer, step
    torch.cuda.empty_cache()
