"""create_model_and_transforms -- drop-in for open_flamingo/src/factory.py:11-119 (same signature and return
triple), building the H100 kernel-backed Flamingo.

Differences forced by the offline / H100-native setting, none of which change the call signature:
  * The vision tower is open_flamingo_b200.src.vit.VisionTransformer (sm_90a kernels).  If `open_clip` is
    importable its pretrained weights and image transform are used (state-dict names are identical); otherwise
    `clip_vision_encoder_path` may be an open_clip model NAME with `clip_vision_encoder_pretrained=None`
    (random init from the built-in config table) or an already-built module exposing `.visual`.
  * `lang_encoder_path` / `tokenizer_path` may be HF hub/local paths (as in the reference) or, for offline use,
    an already-built HF model / a tokenizer-like object with `encode`, `add_special_tokens`, `pad_token`.
"""
from typing import Optional

import torch
from torch import nn

from .flamingo import Flamingo
from .flamingo_lm import FlamingoLMMixin
from .utils import extend_instance
from .vit import CLIPVisionStandIn, VisionTransformer

# vision_cfg of the open_clip model configs Flamingo is used with (open_clip/model_configs/*.json)
_OPEN_CLIP_VISION_CFG = {
    "ViT-L-14": dict(image_size=224, patch_size=14, width=1024, layers=24, heads=16, output_dim=768),
    "ViT-L-14-336": dict(image_size=336, patch_size=14, width=1024, layers=24, heads=16, output_dim=768),
    "ViT-B-16": dict(image_size=224, patch_size=16, width=768, layers=12, heads=12, output_dim=512),
    "ViT-B-32": dict(image_size=224, patch_size=32, width=768, layers=12, heads=12, output_dim=512),
}

# decoder ModuleList attribute per LM family (reference factory.py:132-141)
__KNOWN_DECODER_LAYERS_ATTR_NAMES = {
    "opt": "model.decoder.layers",
    "gptj": "transformer.h",
    "gpt-j": "transformer.h",
    "pythia": "gpt_neox.layers",
    "llama": "model.layers",
    "gptneoxforcausallm": "gpt_neox.layers",
    "mpt": "transformer.blocks",
    "mosaicgpt": "transformer.blocks",
}


def _infer_decoder_layers_attr_name(model):
    cls_name = model.__class__.__name__.lower()
    for key, attr in __KNOWN_DECODER_LAYERS_ATTR_NAMES.items():
        if key.lower() in cls_name:
            return attr
    raise ValueError(
        "We require the attribute name for the nn.ModuleList in the decoder storing the transformer block layers. "
        "Please supply this string manually.")


def _default_image_processor(image_size):
    """CLIP preprocessing as a tensor function (resize to image_size assumed done): (x - mean) / std."""
    mean = torch.tensor([0.48145466, 0.4578275, 0.40821073]).view(3, 1, 1)
    std = torch.tensor([0.26862954, 0.26130258, 0.27577711]).view(3, 1, 1)

    def process(img):
        if not torch.is_tensor(img):
            import numpy as np
            arr = torch.from_numpy(np.asarray(img.convert("RGB").resize((image_size, image_size)))).permute(2, 0, 1)
            img = arr.float() / 255.0
        return (img - mean) / std

    return process


def _build_vision(clip_vision_encoder_path, clip_vision_encoder_pretrained, cache_dir):
    if isinstance(clip_vision_encoder_path, nn.Module):
        enc = clip_vision_encoder_path
        vis = enc.visual if hasattr(enc, "visual") else enc
        wrapped = enc if hasattr(enc, "visual") else CLIPVisionStandIn(enc)
        return wrapped, _default_image_processor(getattr(vis, "image_size", 224)), getattr(vis, "width")
    name = clip_vision_encoder_path
    if clip_vision_encoder_pretrained is not None:
        try:
            import open_clip  # noqa: F401
        except ImportError as e:
            raise ImportError(
                "open_clip is required to load pretrained CLIP weights "
                f"({name!r}, pretrained={clip_vision_encoder_pretrained!r}); install open_clip_torch or pass "
                "clip_vision_encoder_pretrained=None for a randomly initialised tower") from e
        ref_model, _, image_processor = open_clip.create_model_and_transforms(
            name, pretrained=clip_vision_encoder_pretrained, cache_dir=cache_dir)
        cfg = dict(open_clip.get_model_config(name)["vision_cfg"])
        head_width = cfg.get("head_width", 64)
        if head_width != 64:
            raise ValueError(f"{name}: head_width {head_width} (open_clip vision_cfg) is not supported -- the sm_90a "
                             "ViT attention kernel is built for head_dim 64 (ViT-B/L; ViT-H/g/bigG use 80-104)")
        ours = VisionTransformer(image_size=cfg.get("image_size", 224), patch_size=cfg["patch_size"],
                                 width=cfg["width"], layers=cfg["layers"], heads=cfg["width"] // head_width,
                                 mlp_ratio=cfg.get("mlp_ratio", 4.0), output_dim=ref_model.visual.proj.shape[1],
                                 quick_gelu=clip_vision_encoder_pretrained == "openai")
        missing, unexpected = ours.load_state_dict(ref_model.visual.state_dict(), strict=False)
        if missing or unexpected:
            raise KeyError(f"{name}: open_clip visual tower does not match this ViT implementation "
                           f"(missing {sorted(missing)[:4]}, unexpected {sorted(unexpected)[:4]})")
        return CLIPVisionStandIn(ours), image_processor, cfg["width"]
    if name not in _OPEN_CLIP_VISION_CFG:
        raise ValueError(f"unknown CLIP vision config {name!r}; known: {sorted(_OPEN_CLIP_VISION_CFG)}")
    cfg = _OPEN_CLIP_VISION_CFG[name]
    return CLIPVisionStandIn(VisionTransformer(**cfg)), _default_image_processor(cfg["image_size"]), cfg["width"]


def create_model_and_transforms(
    clip_vision_encoder_path,
    clip_vision_encoder_pretrained,
    lang_encoder_path,
    tokenizer_path,
    cross_attn_every_n_layers: int = 1,
    use_local_files: bool = False,
    decoder_layers_attr_name: str = None,
    freeze_lm_embeddings: bool = False,
    cache_dir: Optional[str] = None,
    **flamingo_kwargs,
):
    """Returns (Flamingo model, image processor, tokenizer); see the reference docstring (factory.py:23-41)."""
    vision_encoder, image_processor, vis_dim = _build_vision(clip_vision_encoder_path,
                                                             clip_vision_encoder_pretrained, cache_dir)
    vision_encoder.visual.output_tokens = True  # factory.py:48

    if isinstance(tokenizer_path, str):
        from transformers import AutoTokenizer
        text_tokenizer = AutoTokenizer.from_pretrained(tokenizer_path, local_files_only=use_local_files,
                                                       trust_remote_code=True, cache_dir=cache_dir)
    else:
        text_tokenizer = tokenizer_path
    text_tokenizer.add_special_tokens({"additional_special_tokens": ["<|endofchunk|>", "<image>"]})
    if text_tokenizer.pad_token is None:
        text_tokenizer.add_special_tokens({"pad_token": "<PAD>"})  # labels are masked on pad (train_utils.py:103)

    if isinstance(lang_encoder_path, str):
        from transformers import AutoModelForCausalLM
        lang_encoder = AutoModelForCausalLM.from_pretrained(lang_encoder_path, local_files_only=use_local_files,
                                                            trust_remote_code=True, cache_dir=cache_dir)
        if "mpt-1b-redpajama-200b" in lang_encoder_path:
            # that checkpoint's remote code lacks the embedding accessors (factory.py:72-82)
            class EmbeddingFnMixin:
                def get_input_embeddings(self):
                    return self.transformer.wte

                def set_input_embeddings(self, new_embeddings):
                    self.transformer.wte = new_embeddings

            extend_instance(lang_encoder, EmbeddingFnMixin)
    else:
        lang_encoder = lang_encoder_path

    extend_instance(lang_encoder, FlamingoLMMixin)
    if decoder_layers_attr_name is None:
        decoder_layers_attr_name = _infer_decoder_layers_attr_name(lang_encoder)
    lang_encoder.set_decoder_layers_attr_name(decoder_layers_attr_name)
    lang_encoder.resize_token_embeddings(len(text_tokenizer))

    model = Flamingo(
        vision_encoder,
        lang_encoder,
        text_tokenizer.encode("<|endofchunk|>")[-1],
        text_tokenizer.encode("<image>")[-1],
        vis_dim=vis_dim,
        cross_attn_every_n_layers=cross_attn_every_n_layers,
        **flamingo_kwargs,
    )

    # freeze everything, then unfreeze resampler + gated blocks (+ input embeddings) -- factory.py:104-113
    model.requires_grad_(False)
    assert sum(p.numel() for p in model.parameters() if p.requires_grad) == 0
    model.perceiver.requires_grad_(True)
    model.lang_encoder.gated_cross_attn_layers.requires_grad_(True)
    if not freeze_lm_embeddings:
        model.lang_encoder.get_input_embeddings().requires_grad_(True)
    print(f"Flamingo model initialized with "
          f"{sum(p.numel() for p in model.parameters() if p.requires_grad)} trainable parameters")
    return model, image_processor, text_tokenizer
