"""Flamingo model wrapper: frozen vision encoder -> PerceiverResampler -> gated cross-attention inside a
frozen causal LM.

API parity with the reference's open_flamingo/src/flamingo.py (class Flamingo :17-338): same constructor,
`forward` (:60-122), `generate` (:124-175), `_encode_vision_x` (:177-200), `_condition_media_locations`
(:303-313), `cache_media` / `uncache_media` (:315-338).  `wrap_fsdp` (:202-301) is out of scope: the
data-parallel path replicates the model (OF-3B training fits one 80 GB H100) and all-reduces only the trainable gradients
(see open_flamingo_b200/train.py).
"""
import torch
from torch import nn

from .. import decode_graph
from .helpers import PerceiverResampler


class Flamingo(nn.Module):
    def __init__(self, vision_encoder: nn.Module, lang_encoder: nn.Module, eoc_token_id: int, media_token_id: int,
                 vis_dim: int, cross_attn_every_n_layers: int = 1, gradient_checkpointing: bool = False):
        """
        vision_encoder: CLIP-like object whose `.visual(images)` returns (pooled, tokens)
        lang_encoder:   HF causal LM already extended with FlamingoLMMixin
        eoc_token_id / media_token_id: ids of <|endofchunk|> and <image>
        vis_dim: width of the visual tokens
        """
        super().__init__()
        self.eoc_token_id = eoc_token_id
        self.media_token_id = media_token_id
        self.vis_dim = vis_dim
        cfg = lang_encoder.config
        self.lang_dim = cfg.d_model if hasattr(cfg, "d_model") else cfg.hidden_size  # MPT calls it d_model
        self.vision_encoder = vision_encoder.visual
        self.perceiver = PerceiverResampler(dim=self.vis_dim)
        self.lang_encoder = lang_encoder
        self.lang_encoder.init_flamingo(
            media_token_id=media_token_id,
            lang_hidden_size=self.lang_dim,
            vis_hidden_size=self.vis_dim,
            cross_attn_every_n_layers=cross_attn_every_n_layers,
            gradient_checkpointing=gradient_checkpointing,
        )
        self._use_gradient_checkpointing = gradient_checkpointing
        self.perceiver._use_gradient_checkpointing = gradient_checkpointing
        # the loss returned by forward(labels=...) is HF's shifted causal-LM cross-entropy; route it through the
        # fused kernel pair (falls back to HF's own function for anything but the plain training call)
        if hasattr(type(lang_encoder), "loss_function"):
            from ..fused import causal_lm_loss
            try:
                lang_encoder.loss_function = causal_lm_loss
            except Exception:
                pass

    # ------------------------------------------------------------------ forward
    def forward(self, vision_x: torch.Tensor, lang_x: torch.Tensor, attention_mask: torch.Tensor = None,
                labels: torch.Tensor = None, clear_conditioned_layers: bool = True, past_key_values=None,
                use_cache: bool = False):
        """
        vision_x: (B, T_img, F, C, H, W) with F == 1, or None when media were cached with cache_media()
        lang_x:   (B, T_txt) token ids;  returns the HF CausalLM output (loss first when labels are given)
        """
        lm = self.lang_encoder
        assert lm.initialized_flamingo, "Flamingo layers are not initialized. Please call `init_flamingo` first."
        assert lm._use_cached_vision_x or vision_x is not None, \
            "Must provide either vision_x or have precached media using cache_media()."
        if lm._use_cached_vision_x:
            assert vision_x is None, \
                "Expect vision_x to be None when media has been cached using cache_media(). Try uncache_media() first."
            assert lm.is_conditioned()
        else:
            self._encode_vision_x(vision_x=vision_x)
            self._condition_media_locations(input_ids=lang_x)
        output = lm(input_ids=lang_x, attention_mask=attention_mask, labels=labels,
                    past_key_values=past_key_values, use_cache=use_cache)
        if clear_conditioned_layers:
            lm.clear_conditioned_layers()
        return output

    # ------------------------------------------------------------------ generate
    def generate(self, vision_x: torch.Tensor, lang_x: torch.Tensor, attention_mask: torch.Tensor = None, **kwargs):
        """HF generate() conditioned on images; kwargs are forwarded (max_new_tokens, num_beams, ...).
        Returns lang_x with the generated tokens appended.  When generation uses a cache (`use_cache=True`) under
        bf16 autocast, the frozen MPT and GPT-NeoX blocks decode on the kernels through a kv_cache.KVCache (see
        FlamingoLMMixin.make_kv_cache).  `cache_implementation="static"` (HF's name for a fixed-capacity cache)
        makes that cache fixed-capacity -- prompt plus new tokens, for every beam -- and replays one captured CUDA graph
        per generated token (decode_graph); where the kernels' cache is not made, the argument goes to HF."""
        num_beams = kwargs.pop("num_beams", 1)
        if num_beams > 1:
            vision_x = vision_x.repeat_interleave(num_beams, dim=0)
        lm = self.lang_encoder
        lm._use_cached_vision_x = True
        try:
            self._encode_vision_x(vision_x=vision_x)
            eos_token_id = kwargs.pop("eos_token_id", self.eoc_token_id)
            if kwargs.get("past_key_values") is None and kwargs.get("use_cache", lm.generation_config.use_cache):
                cache = None
                if kwargs.get("cache_implementation") == "static":
                    # HF's precedence: keyword arguments over the call's generation_config over the model's
                    gc = kwargs.get("generation_config") or lm.generation_config
                    capacity = decode_graph.static_cache_capacity(
                        lang_x.shape[1], kwargs.get("max_new_tokens", gc.max_new_tokens),
                        kwargs.get("max_length", gc.max_length))
                    cache = lm.make_kv_cache(capacity=capacity)
                    if cache is not None:
                        kwargs.pop("cache_implementation")
                if cache is None:
                    cache = lm.make_kv_cache()   # bf16 decoding on the kernels; None keeps HF's DynamicCache
                if cache is not None:
                    kwargs["past_key_values"] = cache
            output = lm.generate(input_ids=lang_x, attention_mask=attention_mask, eos_token_id=eos_token_id,
                                 num_beams=num_beams, **kwargs)
        finally:
            lm.clear_conditioned_layers()
            lm._use_cached_vision_x = False
        return output

    # ------------------------------------------------------------------ vision path
    def _encode_vision_x(self, vision_x: torch.Tensor):
        """(B, T_img, F=1, C, H, W) -> ViT tokens (no grad) -> resampler -> condition every decoder layer."""
        assert vision_x.ndim == 6, "vision_x should be of shape (b, T_img, F, C, H, W)"
        b, T, F = vision_x.shape[:3]
        assert F == 1, "Only single frame supported"
        with torch.no_grad():
            tokens = self.vision_encoder(vision_x.reshape(b * T * F, *vision_x.shape[3:]))[1]
        v, d = tokens.shape[1], tokens.shape[2]
        media = self.perceiver(tokens.reshape(b, T, F, v, d))
        for layer in self.lang_encoder._get_decoder_layers():
            layer.condition_vis_x(media)

    def _condition_media_locations(self, input_ids: torch.Tensor):
        media_locations = input_ids == self.media_token_id
        for layer in self.lang_encoder._get_decoder_layers():
            layer.condition_media_locations(media_locations)

    def cache_media(self, input_ids: torch.Tensor, vision_x: torch.Tensor):
        """Pre-compute media for a prompt; later forward() calls (vision_x=None) attend to the LAST image."""
        self._encode_vision_x(vision_x=vision_x)
        self._condition_media_locations(input_ids=input_ids)
        self.lang_encoder._use_cached_vision_x = True

    def uncache_media(self):
        self.lang_encoder.clear_conditioned_layers()
        self.lang_encoder._use_cached_vision_x = False

    def wrap_fsdp(self, *args, **kwargs):
        raise NotImplementedError(
            "FSDP sharding is out of scope for this build: the model is replicated on every GPU; use "
            "open_flamingo_b200.train.FlatTrainer (flat-bucket NCCL all-reduce of the trainable gradients).")
