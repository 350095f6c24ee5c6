"""Graph-replayed decoding: one CUDA graph replay per generated token.

An eager decode step of OF-3B issues about 24 x 40 kernel launches through Python and ctypes, and the GPU waits on that
host work.  With a fixed-capacity kv_cache.KVCache nothing in a one-token step varies on the host: the new token's cache
row and the key count live in a device int32 pair (ops.kv_append, ops.rope_append_dev and ops.attn_decode_dev read
them), the cache buffers never move, and the padding of the keys is a byte buffer beside them.  So the step is captured
once per shape key (batch, capacity, media shape, device) and replayed.  Two LM families are served:

  MPT (OF-3B, OF-9B):   wte(ids) -> per FlamingoLayer: gated block (fused.GatedXattnBlockFn on static media K/V and
                        text_time), then FastMptBlock.decode_step -> norm_f -> lm_head
  GPT-NeoX (OF-4B):     embed_in(ids) -> rotary_emb(h, positions) -> per FlamingoLayer: gated block, then
                        FastNeoXBlock.decode_step -> final_layer_norm -> embed_out

HF's own embedding, rotary module, final norm and output head run under the caller's autocast (with autocast's weight
cache off, so the graph never reads a cast that is freed when the autocast region ends).  MptModel.forward and
GPTNeoXModel.forward are bypassed: their per-call mask construction (and MPT's ALiBi) are not capturable, and the
decoder blocks take their slopes and key mask from elsewhere anyway.  GPT-NeoX's rotary tables come from HF's module run
inside the graph on a static int64 position buffer holding the cache length, the position_ids GPTNeoXModel makes when
the caller passes none: the same torch ops on the same values give the eager step's cos and sin.

Everything the graph reads is a static buffer: ids, the position pair (and GPT-NeoX's position_ids), the new token's
padding byte, the media K/V of every gated layer, text_time, the cache rows and the key mask.  A cache is bound to a
graph by moving its rows into the graph's cache buffers (its first replay in a call); the media inputs are refreshed at
the same time, so one capture serves every later call with the same key.  A call is a run of consecutive replayed steps
on one cache: a step on another cache or media, or after an eager step, a crop or a reset of the cache, starts a new
one.  Every parameter the graph reads is snapshotted as (data_ptr, _version) at capture and checked at the start of
each call; a change (load_state_dict, an optimizer step) re-captures.  A capture that fails leaves that key on the eager
path and keeps the error in `DecodeGraphs.error`.  The replayed step computes what the eager cached step computes, bit
for bit.

The shape key also holds whether inference mode is on: tensors made under `torch.inference_mode` cannot be updated in
place outside it, so a graph whose buffers were made there is never fed under `torch.no_grad`, nor the reverse.

Memory: each key keeps one cache's worth of rows (layers x batch x capacity x 2*H*hd bf16) and its graph's pool for as
long as it is kept (at most MAX_GRAPHS keys per model).  A call's own cache is allocated at its prefill and moved into
those rows at its first replay, so that moment holds two caches.  `lm.decode_graphs.clear()` releases them all.
"""
import collections
import weakref

import torch
from transformers.modeling_outputs import CausalLMOutputWithPast

from . import _lib as L
from . import fused, lm_blocks, ops
from .kv_cache import KVCache, bucket_capacity

MAX_GRAPHS = 4   # captured shape keys kept per model; the least recently used is dropped
# keyword arguments HF's generate and the rank-classification loop pass to a one-token forward
_STEP_KWARGS = {"past_key_values", "use_cache", "return_dict", "output_attentions", "output_hidden_states", "labels",
                "logits_to_keep", "cache_position"}


def static_cache_capacity(prompt_len, max_new_tokens=None, max_length=None):
    """Capacity of the cache of `generate(..., cache_implementation="static")`: the prompt and the new tokens
    (max_new_tokens, else max_length, which counts the prompt, as HF reads them), in bucketed rows.  The batch is HF's
    expanded one (prompts x beams), fixed at the prefill's first write."""
    if max_new_tokens is not None:
        rows = prompt_len + max_new_tokens
    elif max_length is not None:
        rows = max(max_length, prompt_len + 1)
    else:
        raise ValueError("a static cache needs max_new_tokens or max_length")
    return bucket_capacity(rows)


def _autocast_bf16():
    return torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.bfloat16


def _is_neox(lm):
    """A GPT-NeoX LM (HF GPTNeoXForCausalLM); otherwise the LM is taken for an MPT."""
    return hasattr(lm, "gpt_neox")


def _heads(fast):
    """(heads, head_dim) of a decoder block's attention."""
    if isinstance(fast, lm_blocks.FastNeoXBlock):
        a = fast.block.attention
        return a.config.num_attention_heads, a.head_size
    a = fast.block.attn
    return a.n_heads, a.head_dim


def _neox_model_supported(lm):
    """The GPT-NeoX model parts around the blocks are ones the graph replays as GPTNeoXModel.forward runs them: HF's
    default rotary embedding (other rope types, such as dynamic scaling, update their tables from host-side lengths) and
    an embedding dropout that is off."""
    m = lm.gpt_neox
    if not hasattr(lm, "embed_out") or not all(hasattr(m, n) for n in ("embed_in", "rotary_emb", "final_layer_norm")):
        return False
    if getattr(m.rotary_emb, "rope_type", None) != "default":
        return False
    drop = getattr(m, "emb_dropout", None)
    return drop is None or not (drop.training and drop.p > 0)


def eligible(lm, input_ids, attention_mask, cache, use_cached_media, kwargs):
    """True when this forward is a one-token step the graph computes exactly as the eager cached path would.  A
    position_ids keyword (which `generate` does not pass to a Flamingo LM) is one of the calls declined."""
    if not (isinstance(cache, KVCache) and cache.capacity is not None and cache.key_mask_known):
        return False
    if not input_ids.is_cuda or input_ids.dim() != 2 or input_ids.shape[1] != 1 or not use_cached_media:
        return False
    if torch.is_grad_enabled() or not lm_blocks.ENABLED or not _autocast_bf16():
        return False
    if set(kwargs) - _STEP_KWARGS or kwargs.get("labels") is not None or kwargs.get("return_dict") is False:
        return False
    cfg = lm.config
    if kwargs.get("output_attentions", cfg.output_attentions) or \
            kwargs.get("output_hidden_states", cfg.output_hidden_states):
        return False
    B = input_ids.shape[0]
    past = cache.get_seq_length()
    if past < 1 or past + 1 > cache.capacity:
        return False
    if attention_mask is not None and (attention_mask.dim() != 2 or tuple(attention_mask.shape) != (B, past + 1)):
        return False
    if cache.key_mask is None or cache.key_mask.shape[0] != B or cache.key_mask.device != input_ids.device:
        return False
    neox = _is_neox(lm)
    if neox:
        if not _neox_model_supported(lm):
            return False
    elif not all(hasattr(lm, n) for n in ("transformer", "lm_head")) or not hasattr(lm.transformer, "norm_f"):
        return False
    layers = lm._get_decoder_layers()
    if len(layers) != len(cache.layers):
        return False
    for layer, cl in zip(layers, cache.layers):
        fast = getattr(layer, "_fast_block", None)
        if fast is None:
            return False
        if neox:
            # the rotary tables are checked by the capture, once HF's module has made them
            if not isinstance(fast, lm_blocks.FastNeoXBlock) or not fast.block_supported(
                    input_ids, fast.records_outputs(kwargs.get("output_attentions"),
                                                    kwargs.get("output_hidden_states"))):
                return False
            a = fast.block.attention
        else:
            if not fast.supported(input_ids, fast.slopes(input_ids.device), False):
                return False
            a = fast.block.attn
        heads, hd = _heads(fast)
        if a.layer_idx is None or cache.layers[a.layer_idx] is not cl:
            return False
        if not cl.is_initialized or cl.length != past or cl.buf.dtype != torch.bfloat16 or cl.buf.shape[0] != B or \
                cl.buf.device != input_ids.device or cl.heads != heads or cl.head_dim != hd:
            return False
        if layer.gated_cross_attn_layer is not None:
            if layer.vis_x is None or layer.media_locations is None or layer.vis_x.dim() != 4 or \
                    layer.vis_x.shape[0] != B:
                return False
    return True


class _Gated:
    """Static inputs of one gated block."""

    def __init__(self, xattn, B, T_img, n, device):
        a = xattn.attn
        self.xattn = xattn
        self.mode = L.MASK_MEDIA_EQ if a.only_attend_immediate_media else L.MASK_MEDIA_GE
        inner = a.to_q.weight.shape[0]
        self.kv = torch.empty((B * T_img * n, 2 * inner), device=device, dtype=torch.bfloat16)
        self.n = n
        # GatedXattnBlockFn reads only the shape of its media arguments when the media K/V are given
        self.media_shape = torch.empty((B, T_img * n, 0), device=device, dtype=torch.bfloat16)

    def kv_cache(self):
        w = self.xattn.attn.to_kv.weight
        return {(id(w), w._version): self.kv}


class _Entry:
    """One shape key: the captured graph and every buffer it reads."""

    def __init__(self, lm, cache, T_img, n):
        layers = lm._get_decoder_layers()
        B = cache.key_mask.shape[0]
        device = cache.key_mask.device
        # the first bound cache's storage is adopted, unless it was made in the other inference mode
        inference = torch.is_inference_mode_enabled()
        self.bufs = [layer.buf if layer.buf.is_inference() == inference else torch.empty_like(layer.buf)
                     for layer in cache.layers]
        self.key_mask = cache.key_mask if cache.key_mask.is_inference() == inference else \
            torch.empty_like(cache.key_mask)
        self.expect = None   # (cache length, cache.eager_writes) a replay continuing the last one finds
        self.owner = None
        self.media_refs = None
        self.ids = torch.zeros((B, 1), device=device, dtype=torch.int64)
        self.pos_nk = torch.zeros(2, device=device, dtype=torch.int32)
        self.new_masked = torch.zeros(B, device=device, dtype=torch.uint8)
        self.text_time = torch.zeros((B, 1), device=device, dtype=torch.int32)
        self.gated = [None if layer.gated_cross_attn_layer is None else
                      _Gated(layer.gated_cross_attn_layer, B, T_img, n, device) for layer in layers]
        # GPT-NeoX: the position_ids GPTNeoXModel.forward makes for the step, [1, 1] int64 = the cache length
        self.positions = torch.zeros((1, 1), device=device, dtype=torch.int64) if _is_neox(lm) else None
        heads, hd = _heads(layers[0]._fast_block)
        self.workspace = ops.decode_workspace(device, B, heads, hd, cache.capacity)
        self.graph = None
        self.logits = None
        self.failed = False
        self.snapshot = None
        self.keep = ()

    # ---------------------------------------------------------------- binding a cache and the call's media
    def bind(self, cache):
        """Move `cache` onto this entry's buffers (copying its filled rows); the previous owner, if it still uses them,
        gets copies.  Returns True when the binding changed."""
        if self.owner is not None and self.owner() is cache and cache.layers[0].buf is self.bufs[0]:
            return False
        old = self.owner() if self.owner is not None else None
        if old is not None and old is not cache and old.layers[0].buf is self.bufs[0]:
            for layer in old.layers:
                layer.buf = layer.buf.clone()
            old.key_mask = old.key_mask.clone()
        for layer, buf in zip(cache.layers, self.bufs):
            if layer.buf is not buf:
                buf[:, :layer.length].copy_(layer.buf[:, :layer.length])
                layer.buf = buf
        if cache.key_mask is not self.key_mask:
            self.key_mask.copy_(cache.key_mask)
            cache.key_mask = self.key_mask
        self.owner = weakref.ref(cache)
        return True

    def media_changed(self, layer):
        refs = self.media_refs
        return refs is None or refs[0]() is not layer.vis_x or refs[1]() is not layer.media_locations

    def refresh_media(self, layers):
        """Media K/V and text_time of this call, from the media context the eager gated blocks use."""
        from .src.helpers import get_media_context
        first = next((layer for layer in layers if layer.gated_cross_attn_layer is not None), None)
        if first is None:
            return
        ctx = get_media_context(first.vis_x, first.media_locations, True, 1)
        self.text_time.copy_(ctx.text_time)
        M = ctx.media16.shape[0] * ctx.media16.shape[1]
        m2d = ctx.media16.view(M, ctx.media16.shape[2])
        for g in self.gated:
            if g is None:
                continue
            w = g.xattn.attn.to_kv.weight
            key = (id(w), w._version)
            kv = ctx.kv.get(key)
            if kv is None:   # what GatedXattnBlockFn computes and keeps on an eager step
                kv = ops.gemm(m2d, fused.w16(w))
                ctx.kv[key] = kv
            g.kv.copy_(kv)
        self.media_refs = (weakref.ref(first.vis_x), weakref.ref(first.media_locations))

    def set_step(self, input_ids, attention_mask, past):
        self.ids.copy_(input_ids)
        self.pos_nk[0:1].fill_(past)
        self.pos_nk[1:2].fill_(past + 1)
        if self.positions is not None:
            self.positions.fill_(past)
        if attention_mask is None:
            self.new_masked.zero_()
        else:
            self.new_masked.copy_(attention_mask[:, -1] == 0)


def _params(lm):
    """Every parameter a decode step reads (GPT-NeoX: and the rotary module's frequencies)."""
    if _is_neox(lm):
        m = lm.gpt_neox
        ps = list(m.embed_in.parameters()) + list(m.final_layer_norm.parameters()) + list(lm.embed_out.parameters()) + \
            [m.rotary_emb.inv_freq]
    else:
        ps = list(lm.transformer.wte.parameters()) + list(lm.transformer.norm_f.parameters()) + \
            list(lm.lm_head.parameters())
    for layer in lm._get_decoder_layers():
        if layer.gated_cross_attn_layer is not None:
            ps += list(layer.gated_cross_attn_layer.parameters())
        ps += list(layer._fast_block.block.parameters())
    return ps


def _kernel_weights(lm):
    """The parameters whose bf16 copies (fused.w16) the graph reads."""
    ws = []
    # the weights() positions of the GEMM weights: GPT-NeoX query_key_value, dense, dense_h_to_4h, dense_4h_to_h; MPT
    # Wqkv, out_proj, up_proj, down_proj
    gemm = (2, 4, 8, 10) if _is_neox(lm) else (1, 2, 4, 5)
    for layer in lm._get_decoder_layers():
        x = layer.gated_cross_attn_layer
        if x is not None:
            ws += [x.attn.to_q.weight, x.attn.to_out.weight, x.ff[1].weight, x.ff[3].weight]
        w = layer._fast_block.weights()
        ws += [w[i] for i in gemm]
    return ws


def _snapshot(params):
    return [(p.data_ptr(), p._version) for p in params]


class DecodeGraphs:
    """The captured decode steps of one Flamingo LM (FlamingoLMMixin.decode_graphs).  `captures` and `replays` count
    what happened; `error` holds the last capture failure."""

    def __init__(self):
        self.entries = collections.OrderedDict()
        self.captures = 0
        self.replays = 0
        self.error = None
        self._stream = None

    def clear(self):
        """Drop every captured graph with its buffers (caches still using those rows keep them)."""
        self.entries.clear()

    def _body(self, lm, e, cache):
        layers = lm._get_decoder_layers()
        # autocast's weight-cast cache lives until the caller's autocast region ends; a graph must not read from it
        neox = _is_neox(lm)
        with torch.autocast("cuda", dtype=torch.bfloat16, cache_enabled=False):
            if neox:
                m = lm.gpt_neox
                h = m.embed_in(e.ids)
                # GPTNeoXModel.forward's rotary tables, from HF's module on the step's position_ids
                pe = (m.rotary_emb(h, e.positions),)
                if not all(layer._fast_block.supported(h, pe[0], False) for layer in layers):
                    raise ValueError("decode graph: the GPT-NeoX blocks do not take these rotary tables")
            else:
                h = lm.transformer.wte(e.ids)
                pe = ()
            for layer, g, cl in zip(layers, e.gated, cache.layers):
                if g is not None:
                    x = g.xattn
                    a = x.attn
                    h = fused.GatedXattnBlockFn.apply(
                        h.float(), g.media_shape, g.media_shape, e.text_time, g.mode, a.heads, g.n, a.norm.weight,
                        a.norm.bias, a.to_q.weight, a.to_kv.weight, a.to_out.weight, x.attn_gate, x.ff[0].weight,
                        x.ff[0].bias, x.ff[1].weight, x.ff[3].weight, x.ff_gate, g.kv_cache())
                h = layer._fast_block.decode_step(h.float(), cl, e.pos_nk, e.key_mask, e.new_masked, e.workspace, *pe)
            if neox:
                return lm.embed_out(m.final_layer_norm(h))
            return lm.lm_head(lm.transformer.norm_f(h))

    def _capture(self, lm, e, cache):
        cur = torch.cuda.current_stream()
        if self._stream is None or self._stream.device != cur.device:
            self._stream = torch.cuda.Stream(cur.device)
        s = self._stream
        s.wait_stream(cur)
        # one eager step on the capture stream first: kernel attributes, tensor maps, the w16 copies, the slopes and
        # every lazily made buffer come into being outside the capture.  It computes this very step, so it is harmless.
        # It also raises, before any capture, for rotary tables the GPT-NeoX blocks do not take.
        with torch.cuda.stream(s):
            self._body(lm, e, cache)
        cur.wait_stream(s)
        params = _params(lm)
        e.snapshot = _snapshot(params)
        # the graph holds no reference to memory made outside it: keep the weight copies and (MPT) slopes it reads alive
        e.keep = tuple(fused.w16(p) for p in _kernel_weights(lm))
        if not _is_neox(lm):
            e.keep += tuple(layer._fast_block.slopes(e.ids.device) for layer in lm._get_decoder_layers())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            e.logits = self._body(lm, e, cache)
        e.graph = graph
        self.captures += 1

    def step(self, lm, input_ids, attention_mask, cache):
        """Replay the decode step for `input_ids` [B, 1]; returns the model output, or None when this key cannot be
        captured (the caller then runs the eager step)."""
        layers = lm._get_decoder_layers()
        first = next((layer for layer in layers if layer.gated_cross_attn_layer is not None), None)
        T_img, n = (first.vis_x.shape[1], first.vis_x.shape[2]) if first is not None else (0, 0)
        modes = tuple(layer.gated_cross_attn_layer.attn.only_attend_immediate_media for layer in layers
                      if layer.gated_cross_attn_layer is not None)
        key = (input_ids.shape[0], cache.capacity, T_img, n, modes, str(input_ids.device),
               torch.is_inference_mode_enabled())
        e = self.entries.get(key)
        if e is None:
            e = _Entry(lm, cache, T_img, n)
            self.entries[key] = e
            while len(self.entries) > MAX_GRAPHS:
                self.entries.popitem(last=False)
        self.entries.move_to_end(key)
        if e.failed:
            return None
        past = cache.get_seq_length()
        rebound = e.bind(cache)
        if rebound or e.expect != (past, cache.eager_writes) or (first is not None and e.media_changed(first)):
            # the start of a call
            if e.graph is not None and e.snapshot != _snapshot(_params(lm)):
                e.graph, e.logits, e.keep = None, None, ()
            e.refresh_media(layers)
        e.set_step(input_ids, attention_mask, past)
        if e.graph is None:
            try:
                self._capture(lm, e, cache)
            except Exception as ex:   # noqa: BLE001 - any capture failure means: this key stays eager
                self.error = ex
                e.failed = True
                e.graph = None
                torch.cuda.synchronize()
                return None
        e.graph.replay()
        self.replays += 1
        for layer in cache.layers:
            layer.length = past + 1
        e.expect = (past + 1, cache.eager_writes)
        # HF keeps the logits of every step: hand out a copy, never the static buffer
        return CausalLMOutputWithPast(logits=e.logits.clone(), past_key_values=cache)


# kept beside the model rather than on it, so that copying or pickling a model never touches its captured graphs
_GRAPHS = weakref.WeakKeyDictionary()


def graphs_for(lm):
    """The DecodeGraphs of one Flamingo LM, made on first use."""
    graphs = _GRAPHS.get(lm)
    if graphs is None:
        graphs = _GRAPHS[lm] = DecodeGraphs()
    return graphs
