"""Data-parallel training step for the trainable part of Flamingo (resampler + gated cross-attention blocks).

Replaces, for the H100 path, the reference's DDP wrap + clip + AdamW (train/train.py:364-415,
train/train_utils.py:94-216):

  * GradBucket -- ONE flat fp32 gradient buffer for all trainable hot-path parameters, laid out in backward
    completion order (last gated block first, resampler last).  The wgrad GEMM epilogues accumulate straight
    into it (`param._ofk_grad` views, see fused._GradSink), so there is no per-parameter gradient copy and no
    DDP bucket copy.  It is cut into a few contiguous chunks; chunk k's NCCL all-reduce (NVLink 5 / NVSwitch,
    NVLS when available) is launched asynchronously the moment the backward of its last layer has been
    enqueued, so it overlaps the backward of the earlier layers.  Only these gradients are reduced; frozen
    parameters never enter a collective (factory.py:104-113).
  * FlatTrainer -- global-norm clip (train_utils.py:208) and AdamW with the reference's two weight-decay groups
    (decay on `gated_cross_attn` parameters only, train.py:392-408) as one fused kernel per group over the
    flat buffers; the same kernel refreshes the bf16 operand copies the next step's GEMMs read.

The host-side layout/chunking/all-reduce logic is backend-agnostic (gloo on CPU in tests, NCCL on GPUs).
"""
import math

import torch
import torch.distributed as dist

from . import fused, ops

ALIGN = 64  # elements; keeps every parameter view 256-byte (fp32) / 128-byte (bf16) aligned for TMA


def configure_nccl_for_overlap():
    """Call BEFORE torch.distributed.init_process_group(backend="nccl").  Caps the CTAs NCCL uses per collective at the
    number of SMs the persistent GEMM grids leave free while gradient chunks are being reduced (ops.COMM_RESERVED_SMS), so
    the all-reduce kernels run BESIDE the backward GEMMs instead of fighting them for SMs.  Respects an NCCL_MAX_CTAS the
    launcher already set."""
    import os
    if ops.COMM_RESERVED_SMS > 0:
        os.environ.setdefault("NCCL_MAX_CTAS", str(ops.COMM_RESERVED_SMS))


def hot_path_parameters(model):
    """[(name, param)] of the trainable hot-path parameters in backward-completion order."""
    lm = model.lang_encoder
    groups = []
    layers = list(lm.gated_cross_attn_layers)
    for i in reversed(range(len(layers))):
        blk = layers[i]
        if blk is None:
            continue
        ps = [(f"lang_encoder.gated_cross_attn_layers.{i}.{n}", p) for n, p in blk.named_parameters() if p.requires_grad]
        if ps:
            groups.append(("xattn", i, ps))
    per = model.perceiver
    named = [(n, p) for n, p in per.named_parameters() if p.requires_grad]
    if hasattr(per, "layers") and hasattr(per, "norm") and all(hasattr(l, "__getitem__") for l in per.layers):
        # The resampler's backward runs last (its output feeds every gated block) and takes ~2 ms: one group per piece
        # in the order their gradients become final -- final norm, layers depth-1 .. 0, then whatever autograd itself
        # accumulates at the very end (latents, optional frame / media-time embeddings) -- so that only the last,
        # small piece of the all-reduce is exposed after the backward instead of the whole 63 M-parameter resampler.
        taken = set()

        def take(prefix):
            ps = [(f"perceiver.{n}", p) for n, p in named if n.startswith(prefix)]
            taken.update(n for n, _ in named if n.startswith(prefix))
            return ps

        ps = take("norm.")
        if ps:
            groups.append(("perceiver_norm", -1, ps))
        for j in reversed(range(len(per.layers))):
            ps = take(f"layers.{j}.")
            if ps:
                groups.append(("perceiver_layer", j, ps))
        ps = [(f"perceiver.{n}", p) for n, p in named if n not in taken]
        if ps:
            groups.append(("perceiver", -1, ps))
    elif named:
        groups.append(("perceiver", -1, [(f"perceiver.{n}", p) for n, p in named]))
    return groups


def mask_embedding_grad(model, media_token_id=None, endofchunk_token_id=None, rows=None):
    """With trainable LM input embeddings the reference lets only the two ADDED tokens learn: after backward it
    multiplies the embedding gradient by a mask that is one on the `<image>` and `<|endofchunk|>` rows and zero
    elsewhere, before clipping (train_utils.py:172-194).  In place; returns the gradient (or None).  `rows`: optional
    device tensor holding the two row indices (avoids a host-to-device copy, e.g. under CUDA-graph capture)."""
    emb = model.lang_encoder.get_input_embeddings()
    g = emb.weight.grad
    if g is None:
        return None
    media = model.media_token_id if media_token_id is None else media_token_id
    eoc = model.eoc_token_id if endofchunk_token_id is None else endofchunk_token_id
    if rows is None:
        rows = torch.tensor([int(media), int(eoc)], device=g.device)
    keep = g.index_select(0, rows)
    g.zero_()
    g.index_copy_(0, rows, keep)
    return g


class GradBucket:
    """Flat gradient (and optionally parameter) storage with chunked asynchronous all-reduce."""

    def __init__(self, groups, num_chunks=6, process_group=None, flatten_params=True):
        self.pg = process_group
        self.groups = groups
        self.entries = []   # (name, param, offset, numel)
        off = 0
        group_end = []
        for kind, idx, ps in groups:
            for name, p in ps:
                self.entries.append((name, p, off, p.numel()))
                off += (p.numel() + ALIGN - 1) // ALIGN * ALIGN
            group_end.append(off)
        self.total = off
        first = groups[0][2][0][1]
        self.device = first.device
        self.grads = torch.zeros(self.total, device=self.device, dtype=torch.float32)
        self.params = None
        if flatten_params:
            self.params = torch.zeros(self.total, device=self.device, dtype=torch.float32)
        for name, p, o, n in self.entries:
            if flatten_params:
                self.params[o:o + n].view_as(p).copy_(p.data)
                p.data = self.params[o:o + n].view_as(p)
            gview = self.grads[o:o + n].view_as(p)
            p._ofk_grad = gview      # fused wgrad epilogues accumulate here
            p.grad = gview           # anything autograd produces itself (e.g. latents) accumulates in place too
        # chunk boundaries fall on group (layer) ends; the xattn groups are spread over num_chunks-1 chunks and the
        # resampler (whose backward finishes last) is its own chunk.
        xattn_groups = [g for g in range(len(groups)) if groups[g][0] == "xattn"]
        per = max(1, math.ceil(len(xattn_groups) / max(1, num_chunks - 1))) if xattn_groups else 1
        self.chunks = []     # (start, end)
        self.group_to_chunk = {}
        start = 0
        for j, g in enumerate(xattn_groups):
            last_of_chunk = (j + 1) % per == 0 or j == len(xattn_groups) - 1
            self.group_to_chunk[g] = len(self.chunks)
            if last_of_chunk:
                self.chunks.append((start, group_end[g]))
                start = group_end[g]
        # the remaining groups (resampler pieces, in backward-completion order) form two chunks: everything but the last
        # two pieces (final norm, layers depth-1 .. 1) is reduced while layer 0's backward still runs; only layer 0 + the
        # autograd-accumulated leftovers (latents, embeddings) -- a sixth of the resampler -- are reduced after the backward
        rest = [g for g in range(len(groups)) if groups[g][0] != "xattn"]
        parts = [rest[:-2], rest[-2:]] if len(rest) >= 3 else [[g] for g in rest]
        for part in parts:
            if not part:
                continue
            for g in part:
                self.group_to_chunk[g] = len(self.chunks)
            self.chunks.append((start, group_end[part[-1]]))
            start = group_end[part[-1]]
        assert start == self.total
        # any parameter of a block identifies its group from inside the block's backward
        self._param_to_group = {}
        for g, (kind, idx, ps) in enumerate(groups):
            for name, p in ps:
                self._param_to_group[id(p)] = g
        self._chunk_last_group = {}
        for g, c in self.group_to_chunk.items():
            self._chunk_last_group[c] = max(self._chunk_last_group.get(c, -1), g)
        self._pending = []
        self._launched = set()
        self._sync = True      # False inside no_sync(): gradients accumulate locally, nothing is reduced

    # -------------------------------------------------------------- distributed
    @property
    def world(self):
        if not (dist.is_available() and dist.is_initialized()):
            return 1
        return dist.get_world_size(self.pg)

    def zero(self):
        if self._pending:
            raise RuntimeError("GradBucket.zero() with all-reduces still in flight: call finish() / step() first")
        self.grads.zero_()
        self._launched = set()

    def _launch(self, c):
        if c in self._launched:
            return
        self._launched.add(c)
        if self.world > 1:
            s, e = self.chunks[c]
            # While a chunk is being reduced NCCL's CTAs and the persistent GEMM grid compete for SMs: the GEMM tail
            # split (whose owner slice spins on flags written by other clusters of the same grid) is switched off
            # for that window so no GEMM depends on co-residency of all its clusters.
            ops.set_comm_in_flight(True)
            self._pending.append(dist.all_reduce(self.grads[s:e], op=dist.ReduceOp.SUM, group=self.pg, async_op=True))

    def no_sync(self):
        """Context manager for gradient accumulation, with DDP.no_sync()'s meaning: backward passes run inside it
        only ACCUMULATE into the flat buffer; no chunk is reduced.  The reference's optimizer step is several
        backward passes (LAION batch, MMC4 batch, times gradient_accumulation_steps: train_utils.py:109-118,
        :153-172, :206-216); run all but the last one under no_sync() and the chunk all-reduces are launched
        (overlapped with the remaining backward) only during the final backward, when a chunk's contents are final."""
        bucket = self

        class _NoSync:
            def __enter__(self_):
                self_.prev = bucket._sync
                bucket._sync = False

            def __exit__(self_, *exc):
                bucket._sync = self_.prev
                return False

        return _NoSync()

    def on_block_backward_done(self, params):
        """Called by the fused backward of a gated block / resampler layer / final norm once its gradient kernels are
        enqueued (fused.block_backward_hook), with that block's parameter tuple."""
        g = None
        for p in params:
            if p is not None:
                g = self._param_to_group.get(id(p))
                if g is not None:
                    break
        if g is None:
            return
        c = self.group_to_chunk[g]
        if c in self._launched and self.world > 1:
            # a backward pass after this chunk's all-reduce was launched would add local gradients to a buffer that
            # is already (being) reduced: ranks would silently diverge.  Make the mistake loud.
            raise RuntimeError(
                "GradBucket: a backward pass reached a gradient chunk whose all-reduce has already been launched in "
                "this optimizer step.  Run every backward except the last under `trainer.no_sync()` (gradient "
                "accumulation), and call zero_grad() after step().")
        if not self._sync:
            return
        if self._chunk_last_group[c] == g:   # groups complete in increasing g; the chunk's last group closes it
            self._launch(c)

    def finish(self):
        """Launch whatever has not been launched (the resampler chunk) and wait for every all-reduce.
        After this the buffer holds the SUM over ranks (scaling by 1/world is folded into the optimizer)."""
        for c in range(len(self.chunks)):
            self._launch(c)
        for w in self._pending:
            w.wait()
        self._pending = []
        ops.set_comm_in_flight(False)

    def install_hooks(self):
        fused.block_backward_hook = self.on_block_backward_done

    def remove_hooks(self):
        if fused.block_backward_hook == self.on_block_backward_done:
            fused.block_backward_hook = None


class FlatTrainer:
    """zero_grad() -> (user runs forward/backward) -> step().  CUDA only (fused kernels)."""

    def __init__(self, model, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.1, max_grad_norm=1.0,
                 num_chunks=6, process_group=None):
        self.ops = ops
        self.model = model
        self.lr, self.betas, self.eps, self.wd, self.max_norm = lr, betas, eps, weight_decay, max_grad_norm
        groups = hot_path_parameters(model)
        if not groups:
            raise ValueError("model has no trainable resampler / gated cross-attention parameters")
        self.bucket = GradBucket(groups, num_chunks=num_chunks, process_group=process_group)
        b = self.bucket
        self.exp_avg = torch.zeros_like(b.params)
        self.exp_avg_sq = torch.zeros_like(b.params)
        self.w16 = torch.empty(b.total, device=b.device, dtype=torch.bfloat16)
        ops.cast_bf16(b.params, out=self.w16)
        for name, p, o, n in b.entries:
            p._ofk_w16 = self.w16[o:o + n].view(p.shape)
            p._ofk_w16_version = p._version
        # weight-decay segment: the gated blocks come first in the layout (train.py:392-408 decays only them)
        self.decay_end = 0
        ei = 0
        for kind, idx, ps in groups:
            for _ in ps:
                name, p, o, n = b.entries[ei]
                ei += 1
                if kind == "xattn":
                    self.decay_end = o + (n + ALIGN - 1) // ALIGN * ALIGN
        # trainable parameters outside the hot path (LM input embeddings unless frozen): ordinary torch AdamW
        flat_ids = {id(p) for _, p, _, _ in b.entries}
        self.extra = [p for p in model.parameters() if p.requires_grad and id(p) not in flat_ids]
        self.extra_opt = torch.optim.AdamW(self.extra, lr=lr, betas=betas, eps=eps, weight_decay=0.0) if self.extra else None
        emb_w = model.lang_encoder.get_input_embeddings().weight
        self.mask_embeddings = any(p is emb_w for p in self.extra)   # train_utils.py:172-194
        self._embed_rows = torch.tensor([int(model.media_token_id), int(model.eoc_token_id)], device=b.device) \
            if self.mask_embeddings else None
        self.step_count = 0
        # device-resident step counter and learning rate: a captured CUDA graph of the step stays valid as they change
        self.step_dev = torch.zeros(1, device=b.device, dtype=torch.float32)
        self.lr_dev = torch.full((1,), float(lr), device=b.device, dtype=torch.float32)
        self._sumsq = torch.zeros(1, device=b.device, dtype=torch.float32)
        b.install_hooks()

    def zero_grad(self):
        self.bucket.zero()
        for p in self.extra:
            p.grad = None

    def no_sync(self):
        """Gradient accumulation (see GradBucket.no_sync): every backward of an optimizer step except the last."""
        return self.bucket.no_sync()

    def step(self):
        b, ops = self.bucket, self.ops
        b.finish()
        world = b.world
        if self.mask_embeddings:
            mask_embedding_grad(self.model, rows=self._embed_rows)
        if self.extra and world > 1:
            for p in self.extra:
                if p.grad is not None:
                    dist.all_reduce(p.grad, group=b.pg)
        # global grad norm of the MEAN gradient (train_utils.py:208), computed on device, no host sync
        self._sumsq.zero_()
        ops.sumsq_(b.grads, self._sumsq)
        sumsq = self._sumsq
        for p in self.extra:
            if p.grad is not None:
                sumsq = sumsq + p.grad.float().pow(2).sum()
        inv_world = 1.0 / world
        norm = sumsq.sqrt() * inv_world
        clip = torch.clamp(self.max_norm / (norm + 1e-6), max=1.0) * inv_world if self.max_norm else \
            torch.full_like(norm, inv_world)
        clip = clip.float().contiguous()
        self.step_count += 1
        self.step_dev.add_(1.0)
        d = self.decay_end
        if d > 0:
            ops.adamw_(b.params[:d], b.grads[:d], self.exp_avg[:d], self.exp_avg_sq[:d], self.w16[:d], self.lr,
                       self.betas[0], self.betas[1], self.eps, self.wd, self.step_count, clip, self.step_dev,
                       self.lr_dev)
        if d < b.total:
            ops.adamw_(b.params[d:], b.grads[d:], self.exp_avg[d:], self.exp_avg_sq[d:], self.w16[d:], self.lr,
                       self.betas[0], self.betas[1], self.eps, 0.0, self.step_count, clip, self.step_dev, self.lr_dev)
        if self.extra_opt is not None:
            for p in self.extra:
                if p.grad is not None:
                    p.grad.mul_(clip)
            self.extra_opt.step()
        return norm

    def refresh_w16(self):
        """Re-cast every bf16 operand copy from the fp32 masters (fused.w16 also does this lazily, per parameter,
        whenever a parameter's version counter shows it was modified outside the fused optimizer)."""
        self.ops.cast_bf16(self.bucket.params, out=self.w16)
        for name, p, o, n in self.bucket.entries:
            p._ofk_w16_version = p._version

    def set_lr(self, lr):
        """Learning-rate schedule hook (train.py:434-450): updates the host value and the device scalar."""
        self.lr = float(lr)
        self.lr_dev.fill_(float(lr))

    def close(self):
        self.bucket.remove_hooks()


class GraphedTrainStep:
    """Whole training step (zero_grad -> forward under autocast -> backward -> all-reduce -> clip -> AdamW)
    captured ONCE into a CUDA graph and replayed: ~1.5k kernel launches per step collapse into one graph launch,
    removing the inter-kernel launch gaps and all per-step Python/ctypes work.  Inputs are copied into static
    device buffers before each replay.  If capture is impossible (a host synchronisation inside the LM, an
    uncapturable collective, ...) `ok` is False and calls run the same step eagerly."""

    def __init__(self, model, trainer, example_batch, autocast_dtype=torch.bfloat16, warmup=3):
        """example_batch: one batch dict, or a LIST of batch dicts = the micro-batches of one optimizer step (the
        reference's step is a LAION backward + an MMC4 backward, train_utils.py:109-118,153-172): every micro-batch
        but the last runs under trainer.no_sync(), so chunk all-reduces overlap the final backward only."""
        self.model, self.trainer, self.dtype = model, trainer, autocast_dtype
        self.multi = isinstance(example_batch, (list, tuple))
        batches = list(example_batch) if self.multi else [example_batch]
        self.static = [{k: v.clone() for k, v in b.items()} for b in batches]
        self.ok = False
        self.error = None
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):   # also triggers every one-time cudaFuncSetAttribute / cache fill
                self._eager(self.static)
        cur.wait_stream(side)
        torch.cuda.synchronize()
        try:
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.loss = self._eager(self.static)
            self.ok = True
        except Exception as e:   # noqa: BLE001 - any capture failure means: stay eager
            import traceback
            self.error = repr(e)
            self.traceback = traceback.format_exc()
            self.graph = None
            torch.cuda.synchronize()

    def _fwd_bwd(self, batch):
        with torch.autocast("cuda", dtype=self.dtype):
            out = self.model(vision_x=batch["vision_x"], lang_x=batch["lang_x"],
                             attention_mask=batch.get("attention_mask"), labels=batch["labels"])
        out.loss.backward()
        return out.loss.detach()

    def _eager(self, batches):
        self.trainer.zero_grad()
        loss = None
        for i, batch in enumerate(batches):
            if i + 1 < len(batches):
                with self.trainer.no_sync():
                    l = self._fwd_bwd(batch)
            else:
                l = self._fwd_bwd(batch)
            loss = l if loss is None else loss + l
        self.trainer.step()
        return loss

    def __call__(self, batch):
        batches = list(batch) if self.multi else [batch]
        if not self.ok:
            return self._eager(batches)
        for st, b in zip(self.static, batches):
            for k, v in b.items():
                if v is not st[k]:
                    st[k].copy_(v, non_blocking=True)
        self.graph.replay()
        return self.loss
