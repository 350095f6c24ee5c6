"""Language-model side of Flamingo: the per-layer wrapper and the mixin spliced onto a HF causal LM.

Interface parity with the reference's open_flamingo/src/flamingo_lm.py:
  FlamingoLayer  (:6-66)   -- gated cross-attention block (or None) in front of one frozen decoder block
  FlamingoLMMixin (:69-167) -- init_flamingo / forward / is_conditioned / clear_conditioned_layers, plus the
                               `gated_cross_attn_layers` and `old_decoder_blocks` attributes whose names
                               appear in released checkpoints (train_utils.py:321-330).
The gated blocks are the kernel-backed ones from .helpers; the decoder blocks stay the frozen LM's own
PyTorch modules.
"""
import torch
import torch.nn as nn

from .. import decode_graph, lm_blocks
from ..kv_cache import KVCache
from .helpers import GatedCrossAttentionBlock
from .utils import getattr_recursive, setattr_recursive


class FlamingoLayer(nn.Module):
    """One decoder position: optional gated cross-attention block, then the frozen decoder block
    (flamingo_lm.py:6-66).  State set from outside before each forward, exactly as in the reference:
      vis_x            (B, T_img, n_latents, D_vis) resampler output, shared by all layers (`condition_vis_x`)
      media_locations  (B, T_txt) bool, True at `<image>` tokens (`condition_media_locations`)
      use_cached_media bool, decode-time switch: every text token attends the last cached image
    The attribute names `gated_cross_attn_layer` / `decoder_layer` are part of the checkpoint key names."""

    def __init__(self, gated_cross_attn_layer, decoder_layer, gradient_checkpointing=False):
        super().__init__()
        self.gated_cross_attn_layer = gated_cross_attn_layer
        self.decoder_layer = decoder_layer
        self.vis_x = None
        self.media_locations = None
        self.use_cached_media = None
        # recognised frozen decoder blocks (HF MptBlock, GPTNeoXLayer, LlamaDecoderLayer, OPTDecoderLayer) run on the sm_90a
        # kernels; everything else -- and every case the fast path declines -- runs the block's own PyTorch forward as
        # in the reference
        self._fast_block = lm_blocks.accelerate(decoder_layer)
        self._pure_causal_flag = None
        # kept for API compatibility (train.py:368-381); the fused blocks already store only what backward needs
        if gated_cross_attn_layer is not None:
            gated_cross_attn_layer._use_gradient_checkpointing = gradient_checkpointing
        decoder_layer._use_gradient_checkpointing = gradient_checkpointing

    def is_conditioned(self) -> bool:
        """True once both the visual features and the media locations are in place (flamingo_lm.py:28-30)."""
        return self.vis_x is not None and self.media_locations is not None

    # the three setters below are called per forward by Flamingo / FlamingoLMMixin (flamingo_lm.py:33-41)
    def condition_vis_x(self, vis_x):
        self.vis_x = vis_x

    def condition_media_locations(self, media_locations):
        self.media_locations = media_locations

    def condition_use_cached_media(self, use_cached_media):
        self.use_cached_media = use_cached_media

    def forward(self, lang_x, attention_mask=None, **decoder_layer_kwargs):
        """lang_x (B, T_txt, D) -> whatever the wrapped decoder block returns (flamingo_lm.py:43-66).  The gated
        block runs on libofk (fused.GatedXattnBlockFn); a recognised frozen block too (lm_blocks.FrozenMptBlockFn,
        FrozenNeoXBlockFn), falling back to the block's own PyTorch forward whenever the fast path declines (KV cache,
        dropout, ...)."""
        xattn = self.gated_cross_attn_layer
        if xattn is not None:
            # same failure modes as the reference (flamingo_lm.py:47-53)
            if self.vis_x is None:
                raise ValueError("vis_x must be conditioned before forward pass")
            if self.media_locations is None:
                raise ValueError("media_locations must be conditioned before forward pass")
            lang_x = xattn(lang_x, self.vis_x, media_locations=self.media_locations,
                           use_cached_media=self.use_cached_media)
        if self._fast_block is not None:
            res = self._fast_block(lang_x, attention_mask=attention_mask, pure_causal_flag=self._pure_causal_flag,
                                   **decoder_layer_kwargs)
            if res is not None:
                return res
        return self.decoder_layer(lang_x, attention_mask=attention_mask, **decoder_layer_kwargs)


class FlamingoLMMixin(nn.Module):
    """Mixed into a HF causal LM instance with utils.extend_instance (factory.py:85)."""

    def set_decoder_layers_attr_name(self, decoder_layers_attr_name):
        """Dotted path of the decoder's nn.ModuleList inside the HF model, e.g. "transformer.blocks" for MPT
        (factory.py:86,132-141)."""
        self.decoder_layers_attr_name = decoder_layers_attr_name

    def _get_decoder_layers(self):
        return getattr_recursive(self, self.decoder_layers_attr_name)

    def _set_decoder_layers(self, value):
        setattr_recursive(self, self.decoder_layers_attr_name, value)

    def init_flamingo(self, media_token_id, lang_hidden_size, vis_hidden_size, cross_attn_every_n_layers,
                      gradient_checkpointing):
        """Insert a gated block before every n-th decoder block: block i gets one iff (i + 1) % n == 0
        (flamingo_lm.py:100)."""
        blocks = self._get_decoder_layers()
        self.old_decoder_blocks = blocks
        every = cross_attn_every_n_layers
        self.gated_cross_attn_layers = nn.ModuleList([
            GatedCrossAttentionBlock(dim=lang_hidden_size, dim_visual=vis_hidden_size) if (i + 1) % every == 0 else None
            for i in range(len(blocks))
        ])
        self.init_flamingo_layers(gradient_checkpointing)
        self.media_token_id = media_token_id
        self.initialized_flamingo = True
        self._use_cached_vision_x = False

    def init_flamingo_layers(self, gradient_checkpointing):
        """(Re)build the FlamingoLayer list from gated_cross_attn_layers / old_decoder_blocks."""
        pairs = zip(self.gated_cross_attn_layers, self.old_decoder_blocks)
        self._set_decoder_layers(nn.ModuleList([FlamingoLayer(x, blk, gradient_checkpointing) for x, blk in pairs]))

    def forward(self, input_ids, attention_mask, **kwargs):
        """Derive media_locations from the ids, push the conditioning into every layer, then run the HF model's own
        forward (flamingo_lm.py:127-155).  Additions that do not change results: the device-side all-ones flag for
        the attention kernel and the capture-safe 4-D mask (see below)."""
        if not getattr(self, "initialized_flamingo", False):
            raise ValueError("Flamingo layers are not initialized. Please call `init_flamingo` first.")
        if kwargs.get("use_cache") and kwargs.get("past_key_values") is None:
            cache = self.make_kv_cache()   # a cached prefix (rank classification): decode its continuation on the kernels
            if cache is not None:
                kwargs["past_key_values"] = cache
        cache = kwargs.get("past_key_values")
        fixed = isinstance(cache, KVCache) and cache.capacity is not None
        if fixed:
            cache.check_room(input_ids.shape[1])   # before any work is queued
        media_locations = input_ids == self.media_token_id
        # HF generate() feeds one token at a time after the prompt; such calls carry no <image> token and must
        # keep attending to the last cached image (flamingo_lm.py:137-146).
        use_cached = bool(self._use_cached_vision_x and self.is_conditioned() and not media_locations.any())
        for layer in self._get_decoder_layers():
            if not use_cached:
                layer.condition_media_locations(media_locations)
            layer.condition_use_cached_media(use_cached)
        if fixed:
            # a fixed-capacity cache: one-token steps replay a captured CUDA graph (decode_graph); any other step runs
            # eagerly on the same buffers
            if decode_graph.eligible(self, input_ids, attention_mask, cache, use_cached, kwargs):
                out = self.decode_graphs.step(self, input_ids, attention_mask, cache)
                if out is not None:
                    return out
            cache.note_key_padding(attention_mask, input_ids.shape[0], input_ids.shape[1], input_ids.device)
        # device-side "attention_mask is all ones" flag: lets the LM attention kernel take its pure-causal fast path
        # without a host synchronisation
        if input_ids.is_cuda:
            flag = torch.ones(1, dtype=torch.int32, device=input_ids.device) if attention_mask is None else \
                attention_mask.all().to(torch.int32).reshape(1)
        else:
            flag = None
        for layer in self._get_decoder_layers():
            layer._pure_causal_flag = flag
        if input_ids.is_cuda and torch.cuda.is_current_stream_capturing() and type(self).__mro__[2].__name__.startswith("Mpt") \
                and (attention_mask is None or attention_mask.dim() == 2) and kwargs.get("past_key_values") is None:
            # CUDA-graph capture: HF's mask builder creates a device scalar from a Python float (an unpinned H2D
            # copy, illegal while capturing).  Hand the MPT body the finished 4-D mask instead -- same content:
            # True = masked = (key after query) | (key is padding); HF returns a 4-D mask unchanged.
            T = input_ids.shape[1]
            future = torch.ones(T, T, dtype=torch.bool, device=input_ids.device).triu(1)
            m4 = future.view(1, 1, T, T).expand(input_ids.shape[0], 1, T, T)
            if attention_mask is not None:
                m4 = m4 | (attention_mask == 0).view(input_ids.shape[0], 1, 1, T)
            attention_mask = m4.contiguous()
        elif input_ids.is_cuda and torch.cuda.is_current_stream_capturing() and \
                type(self).__mro__[2].__name__.startswith("OPT") and attention_mask is not None and \
                attention_mask.dim() == 2 and kwargs.get("past_key_values") is None and kwargs.get("position_ids") is None:
            # The same for OPT, whose decoder also derives its learned positions from the 2-D mask: hand it those
            # positions (OPTDecoder's own formula) and the 4-D mask in its sdpa form, True = attend =
            # (key not after query) & (key is not padding).
            B, T = input_ids.shape
            kwargs["position_ids"] = (torch.cumsum(attention_mask, dim=1) * attention_mask - 1).long()
            causal = torch.ones(T, T, dtype=torch.bool, device=input_ids.device).tril()
            attention_mask = (causal.view(1, 1, T, T) & (attention_mask != 0).view(B, 1, 1, T)).contiguous()
        return super().forward(input_ids=input_ids, attention_mask=attention_mask, **kwargs)

    def make_kv_cache(self, capacity=None):
        """A kv_cache.KVCache for decoding this LM on the kernels, or None where HF's own cache is kept: it is made only
        on CUDA, under `torch.autocast("cuda", dtype=torch.bfloat16)` (the caller asked for bf16 numerics; the cache
        stores bf16), with lm_blocks.ENABLED, and when every decoder block is a recognised MPT, GPT-NeoX, LLaMA or OPT block.  In
        fp32 every path stays HF's.

        capacity: None for a cache that grows; an int for a fixed-capacity cache of at least that many rows, with which
        `forward(..., past_key_values=cache)` replays one captured CUDA graph per one-token step (decode_graph).  Its
        buffers are allocated at the first write; each captured shape also keeps a cache's worth of rows until
        `self.decode_graphs.clear()`."""
        if not lm_blocks.ENABLED or not torch.is_autocast_enabled("cuda") or \
                torch.get_autocast_dtype("cuda") != torch.bfloat16:
            return None
        layers = self._get_decoder_layers()
        if not all(isinstance(layer, FlamingoLayer) and layer._fast_block is not None for layer in layers):
            return None
        if not self.get_input_embeddings().weight.is_cuda:
            return None
        return KVCache(len(layers), capacity=capacity)

    @property
    def decode_graphs(self):
        """The captured decode steps of this model (decode_graph.DecodeGraphs), made on first use."""
        return decode_graph.graphs_for(self)

    def is_conditioned(self) -> bool:
        """All layers hold vis_x and media_locations (flamingo_lm.py:157-159)."""
        return all(layer.is_conditioned() for layer in self._get_decoder_layers())

    def clear_conditioned_layers(self):
        """Drop the per-forward state of every layer (flamingo_lm.py:161-167); Flamingo.forward calls this unless
        `clear_conditioned_layers=False` (media cached for scoring, flamingo.py:118-119)."""
        for layer in self._get_decoder_layers():
            layer.condition_vis_x(None)
            layer.condition_media_locations(None)
            layer.condition_use_cached_media(None)
