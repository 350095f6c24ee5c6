"""KV cache of the frozen MPT blocks in the layout the attention kernels read.

HF's `DynamicCache` keeps K and V as separate `[B, H, T, hd]` tensors and `torch.cat`s every new token onto them, which
rewrites the whole cache on every decode step.  `KVCache` keeps, per layer, one buffer `[B, capacity, 2*H*hd]`: the K
columns, then the V columns, one row per position -- the column-slice layout of the qkv projection.  The dense and
decode attention kernels read K and V as strided views of it (row stride 2*H*hd) without a copy, and the cached fast
path of lm_blocks.FastMptBlock writes new rows straight into it from the K/V projection GEMM.

It is a `transformers.Cache`, so HF's `generate` (greedy, sampling, beam search), `create_causal_mask` and a block that
takes HF's own `MptAttention` use it unchanged through `update()`, which takes and returns HF's `[B, H, T, hd]` layout.
The sequence length is tracked on the host, so `get_seq_length` never reads the device.  Capacity grows geometrically
and a growth copies only the filled rows.
"""
import torch
from transformers.cache_utils import Cache, CacheLayerMixin

_ROW_ALIGN = 16   # capacity granularity, in rows


class KVCacheLayer(CacheLayerMixin):
    is_sliding = False

    def __init__(self):
        super().__init__()
        self.buf = None   # [B, capacity, 2 * H * hd]; K columns [0, H*hd), V columns [H*hd, 2*H*hd)
        self.length = 0
        self.heads = self.head_dim = 0

    def lazy_initialization(self, key_states, value_states=None):
        B, H, _, hd = key_states.shape
        self.init_storage(B, H, hd, key_states.dtype, key_states.device)

    def init_storage(self, batch, heads, head_dim, dtype, device):
        """First write: fixes the batch, head layout and storage dtype (bf16 under autocast)."""
        self.heads, self.head_dim = heads, head_dim
        self.dtype, self.device = dtype, device
        self.buf = torch.empty((batch, 0, 2 * heads * head_dim), dtype=dtype, device=device)
        self.length = 0
        self.is_initialized = True

    @property
    def capacity(self):
        return 0 if self.buf is None else self.buf.shape[1]

    def reserve(self, n):
        """Make room for `n` more rows; returns the buffer.  Growth doubles the capacity and copies rows [0, length)."""
        need = self.length + n
        if need > self.capacity:
            cap = -(-max(need, 2 * self.capacity) // _ROW_ALIGN) * _ROW_ALIGN
            B, _, W = self.buf.shape
            buf = torch.empty((B, cap, W), dtype=self.buf.dtype, device=self.buf.device)
            if self.length:
                buf[:, :self.length].copy_(self.buf[:, :self.length])
            self.buf = buf
        return self.buf

    def kv_views(self):
        """K and V of rows [0, length) as [B, length, H*hd] views of the buffer."""
        D = self.heads * self.head_dim
        rows = self.buf[:, :self.length]
        return rows[..., :D], rows[..., D:]

    def update(self, key_states, value_states, *args, **kwargs):
        """Append `[B, H, T, hd]` keys and values; returns all cached keys and values as contiguous tensors in the same
        layout (what DynamicCache returns, so HF's attention computes exactly what it computes with DynamicCache)."""
        if not self.is_initialized:
            self.lazy_initialization(key_states, value_states)
        B, H, T, hd = key_states.shape
        D = H * hd
        buf = self.reserve(T)
        rows = buf[:, self.length:self.length + T]
        rows[..., :D].copy_(key_states.transpose(1, 2).reshape(B, T, D))
        rows[..., D:].copy_(value_states.transpose(1, 2).reshape(B, T, D))
        self.length += T
        k, v = self.kv_views()
        return (k.reshape(B, self.length, H, hd).transpose(1, 2).contiguous(),
                v.reshape(B, self.length, H, hd).transpose(1, 2).contiguous())

    def get_mask_sizes(self, query_length):
        return self.length + query_length, 0

    def get_seq_length(self):
        return self.length

    def get_max_cache_shape(self):
        return -1

    def reorder_cache(self, beam_idx):
        if self.length > 0:
            self.buf = self.buf.index_select(0, beam_idx.to(self.buf.device))

    def crop(self, max_length):
        if max_length < 0:
            max_length = self.length + max_length
        self.length = max(0, min(self.length, max_length))

    def reset(self):
        self.length = 0


class KVCache(Cache):
    """One KVCacheLayer per decoder block (the block's `attn.layer_idx`)."""

    def __init__(self, num_layers):
        super().__init__(layers=[KVCacheLayer() for _ in range(num_layers)])
