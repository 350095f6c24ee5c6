"""GPU: the data-parallel training step machinery (train.FlatTrainer / GraphedTrainStep) -- flat-bucket gradients,
fused clip + AdamW with the reference's weight-decay groups (train.py:392-408), and the CUDA-graphed step."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

VIT = dict(image_size=56, patch_size=14, width=128, layers=2, heads=2, output_dim=128)
MPT = dict(d_model=128, n_heads=2, n_layers=2, vocab_size=61, max_seq_len=64, expansion_ratio=2)


def build(seed=0):
    from open_flamingo_b200.testing import build_flamingo, synthetic_batch
    model, _, tok = build_flamingo(VIT, MPT, device="cuda", gate_init=1.0, seed=seed)
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    batch = {k: v.cuda() for k, v in synthetic_batch(3, 2, 24, media_id, eoc_id, 61, image_size=56, seed=9).items()}
    return model.train(), batch


def fwd_bwd(model, batch):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = model(vision_x=batch["vision_x"], lang_x=batch["lang_x"], attention_mask=batch["attention_mask"],
                    labels=batch["labels"])
    out.loss.backward()
    return out.loss.detach()


def test_flat_trainer_matches_torch_adamw_with_clip():
    from open_flamingo_b200.train import FlatTrainer
    model, batch = build()
    ref = copy.deepcopy(model)
    # --- reference semantics: clip_grad_norm_(1.0) then AdamW, decay only on gated_cross_attn params
    named = [(n, p) for n, p in ref.named_parameters() if p.requires_grad]
    decay = [p for n, p in named if "gated_cross_attn" in n]
    rest = [p for n, p in named if "gated_cross_attn" not in n]
    opt = torch.optim.AdamW([{"params": decay, "weight_decay": 0.1}, {"params": rest, "weight_decay": 0.0}], lr=1e-3)
    trainer = FlatTrainer(model, lr=1e-3, weight_decay=0.1, max_grad_norm=1.0)
    got = dict(model.named_parameters())
    for _ in range(3):
        trainer.zero_grad()
        fwd_bwd(model, batch)
        # hand the SAME gradients to the torch optimizer (Adam turns noise-level gradient differences into +-lr
        # parameter differences, so the two optimizers must see identical inputs to be compared tightly)
        for n, p in named:
            p.grad = got[n].grad.detach().clone()
        torch.nn.utils.clip_grad_norm_([p for _, p in named], 1.0)
        opt.step()
        trainer.step()
    for n, p in named:
        err = (got[n].detach() - p.detach()).abs().max().item()
        assert err <= 2e-6 + 1e-5 * p.detach().abs().max().item(), f"{n}: {err}"
    # parameters keep their reference names and now live in the flat buffer
    assert got["perceiver.latents"].data_ptr() >= trainer.bucket.params.data_ptr()


def test_graphed_step_equals_eager_step():
    from open_flamingo_b200.train import FlatTrainer, GraphedTrainStep
    m1, batch = build(seed=1)
    m2 = copy.deepcopy(m1)
    t1 = FlatTrainer(m1, lr=1e-3)
    losses_eager = []
    for _ in range(4):
        t1.zero_grad()
        losses_eager.append(fwd_bwd(m1, batch).item())
        t1.step()
    t1.close()
    t2 = FlatTrainer(m2, lr=1e-3)
    g = GraphedTrainStep(m2, t2, batch, warmup=1)
    assert g.ok, g.error
    # warm-up consumed 1 eager step and the capture itself does not execute: replays continue from step 2
    losses_graph = [losses_eager[0]] + [g(batch).item() for _ in range(3)]
    for a, b in zip(losses_eager[1:], losses_graph[1:]):
        assert abs(a - b) <= 2e-2 * abs(a) + 1e-3, (losses_eager, losses_graph)
    # a different batch through the same graph (static input buffers are refreshed)
    b2 = {k: v.clone() for k, v in batch.items()}
    b2["vision_x"] = torch.randn_like(b2["vision_x"])
    l_new = g(b2).item()
    assert l_new == l_new and abs(l_new - losses_graph[-1]) > 0


def test_trainable_embeddings_only_update_the_two_added_tokens():
    """freeze_lm_embeddings=False (the reference default): the embedding gradient is masked to the <image> and
    <|endofchunk|> rows before clipping (train_utils.py:172-194), so every other row must stay bit-identical."""
    from open_flamingo_b200.testing import build_flamingo, synthetic_batch
    from open_flamingo_b200.train import FlatTrainer
    model, _, tok = build_flamingo(VIT, MPT, device="cuda", gate_init=1.0, seed=3, freeze_lm_embeddings=False)
    model.train()
    media_id, eoc_id = tok.encode("<image>")[-1], tok.encode("<|endofchunk|>")[-1]
    batch = {k: v.cuda() for k, v in synthetic_batch(3, 2, 24, media_id, eoc_id, 61, image_size=56, seed=9).items()}
    emb = model.lang_encoder.get_input_embeddings().weight
    assert emb.requires_grad
    before = emb.detach().clone()
    trainer = FlatTrainer(model, lr=1e-2, weight_decay=0.1, max_grad_norm=1.0)
    assert trainer.mask_embeddings
    for _ in range(2):
        trainer.zero_grad()
        fwd_bwd(model, batch)
        trainer.step()
    changed = (emb.detach() != before).any(1).nonzero().flatten().tolist()
    assert changed == sorted([media_id, eoc_id]), changed


def test_checkpoint_resume_continues_the_same_trajectory(tmp_path):
    """save_checkpoint / load_checkpoint (reference format, train_utils.py:337-375 / train.py:297-308) restore
    parameters, flat AdamW moments, step count and the bf16 operand copies: the step after a resume reproduces
    the step of the uninterrupted run."""
    import os
    from open_flamingo_b200.checkpoint import load_checkpoint, save_checkpoint
    from open_flamingo_b200.train import FlatTrainer
    m1, batch = build(seed=4)
    t1 = FlatTrainer(m1, lr=1e-3, weight_decay=0.1, max_grad_norm=1.0)
    for _ in range(2):
        t1.zero_grad()
        fwd_bwd(m1, batch)
        t1.step()
    path = os.path.join(tmp_path, "checkpoint_0.pt")
    save_checkpoint(path, m1, t1, epoch=0)
    t1.zero_grad()
    l_ref = fwd_bwd(m1, batch)
    t1.step()
    t1.zero_grad()
    l_ref2 = fwd_bwd(m1, batch)

    m2, _ = build(seed=4)
    with torch.no_grad():                                   # start from different weights: everything must come from disk
        for p in m2.parameters():
            if p.requires_grad:
                p.add_(0.05)
    t2 = FlatTrainer(m2, lr=1e-3, weight_decay=0.1, max_grad_norm=1.0)
    assert load_checkpoint(path, m2, t2) == 1
    assert t2.step_count == 2
    t2.zero_grad()
    l_new = fwd_bwd(m2, batch)
    t2.step()
    t2.zero_grad()
    l_new2 = fwd_bwd(m2, batch)
    assert abs(l_new.item() - l_ref.item()) <= 1e-4 * abs(l_ref.item()), (l_new.item(), l_ref.item())
    assert abs(l_new2.item() - l_ref2.item()) <= 2e-3 * abs(l_ref2.item()), (l_new2.item(), l_ref2.item())


def test_training_step_is_bitwise_reproducible():
    """Two copies of one model, trained on the same batch, end every step with bit-identical loss, gradients and
    parameters: no reduction in the step may depend on the order in which CTAs finish (Adam would turn such last-bit
    noise in near-zero gradient entries into parameter changes of up to the learning rate)."""
    from open_flamingo_b200.train import FlatTrainer
    m1, batch = build(seed=2)
    m2 = copy.deepcopy(m1)
    t1, t2 = FlatTrainer(m1, lr=1e-3), FlatTrainer(m2, lr=1e-3)
    for step in range(3):
        losses = []
        for m, t in ((m1, t1), (m2, t2)):
            t.zero_grad()
            losses.append(fwd_bwd(m, batch))
            t.step()
        torch.cuda.synchronize()
        assert torch.equal(losses[0], losses[1]), (step, losses)
        assert torch.equal(t1.bucket.grads, t2.bucket.grads), f"step {step}: gradients differ"
        assert torch.equal(t1.bucket.params, t2.bucket.params), f"step {step}: parameters differ"
