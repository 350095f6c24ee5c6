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

`KVCache(num_layers, capacity=n)` is a fixed-capacity cache instead: every layer's buffer holds `n` rows rounded up to
a multiple of CAPACITY_BUCKET and is allocated once, with one `[B, round_up(capacity, 8)]` byte buffer beside them that
marks the padding keys (nonzero = masked).  Its buffers never move -- an overflow raises, beam search permutes rows in
place, crop and reset only move the host length -- which is what lets decode_graph replay one captured CUDA graph for
every decode step.  It serves HF's and the kernels' eager paths exactly as the growing cache does.
"""
import torch
from transformers.cache_utils import Cache, CacheLayerMixin

_ROW_ALIGN = 16   # capacity granularity of a growing cache, in rows
# a fixed capacity is rounded up to a multiple of this, so that prompts of similar length share one captured graph
CAPACITY_BUCKET = 64


def bucket_capacity(rows):
    """The capacity a fixed-capacity cache asked for `rows` rows gets."""
    if rows < 1:
        raise ValueError(f"a fixed-capacity KV cache needs a capacity >= 1, got {rows}")
    return -(-rows // CAPACITY_BUCKET) * CAPACITY_BUCKET


class KVCacheLayer(CacheLayerMixin):
    is_sliding = False

    def __init__(self, fixed_capacity=None):
        super().__init__()
        self.buf = None   # [B, capacity, 2 * H * hd]; K columns [0, H*hd), V columns [H*hd, 2*H*hd)
        self.length = 0
        self.heads = self.head_dim = 0
        self.fixed_capacity = fixed_capacity

    def lazy_initialization(self, key_states, value_states=None):
        B, H, _, hd = key_states.shape
        self.init_storage(B, H, hd, key_states.dtype, key_states.device)

    def init_storage(self, batch, heads, head_dim, dtype, device):
        """First write: fixes the batch, head layout and storage dtype (bf16 under autocast)."""
        self.heads, self.head_dim = heads, head_dim
        self.dtype, self.device = dtype, device
        rows = self.fixed_capacity or 0
        self.buf = torch.empty((batch, rows, 2 * heads * head_dim), dtype=dtype, device=device)
        self.length = 0
        self.is_initialized = True

    @property
    def capacity(self):
        return 0 if self.buf is None else self.buf.shape[1]

    def reserve(self, n):
        """Make room for `n` more rows; returns the buffer.  Growth doubles the capacity and copies rows [0, length).
        A fixed-capacity layer never grows: it raises ValueError instead."""
        need = self.length + n
        if self.fixed_capacity is not None and need > self.fixed_capacity:
            raise ValueError(f"KV cache overflow: {need} rows needed, capacity {self.fixed_capacity}")
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
            if self.fixed_capacity is None:
                self.buf = self.buf.index_select(0, beam_idx.to(self.buf.device))
            else:   # in place: the buffer's address is part of a captured decode graph
                rows = self.buf[:, :self.length]
                rows.copy_(rows.index_select(0, beam_idx.to(self.buf.device)))

    def crop(self, max_length):
        if max_length < 0:
            max_length = self.length + max_length
        self.length = max(0, min(self.length, max_length))

    def reset(self):
        self.length = 0


class KVCache(Cache):
    """One KVCacheLayer per decoder block (the block's `attn.layer_idx`).  capacity=None: each layer grows as needed;
    an int: a fixed-capacity cache of bucket_capacity(capacity) rows (see the module docstring)."""

    def __init__(self, num_layers, capacity=None):
        self.capacity = None if capacity is None else bucket_capacity(int(capacity))
        super().__init__(layers=[KVCacheLayer(self.capacity) for _ in range(num_layers)])
        self.key_mask = None   # fixed capacity: [B, round_up(capacity, 8)] uint8, nonzero = padding key
        self.key_mask_known = True   # False once a step came with a mask other than HF's 2-D one
        # counts eager appends, crops and resets: a graph-replayed step knows from it whether it continues the last one
        self.eager_writes = 0

    def ensure_key_mask(self, batch, device):
        if self.key_mask is None or self.key_mask.shape[0] != batch or self.key_mask.device != torch.device(device):
            self.key_mask = torch.zeros((batch, -(-self.capacity // 8) * 8), dtype=torch.uint8, device=device)
        return self.key_mask

    def check_room(self, n):
        """Raise ValueError, before any work is queued, if `n` more rows do not fit a fixed-capacity cache."""
        if self.capacity is not None and self.get_seq_length() + n > self.capacity:
            raise ValueError(f"KV cache overflow: {self.get_seq_length() + n} rows needed, capacity {self.capacity}")

    def note_key_padding(self, attention_mask, batch, n, device):
        """Record the padding of the `n` rows about to be appended from HF's 2-D attention mask (1 = token,
        0 = padding; None = no padding).  Any other mask leaves the key mask unknown until reset()."""
        past = self.get_seq_length()
        mask = self.ensure_key_mask(batch, device)
        self.eager_writes += 1
        if attention_mask is None:
            mask[:, past:past + n].zero_()
        elif attention_mask.dim() == 2 and attention_mask.shape[0] == batch and attention_mask.shape[1] >= n:
            mask[:, past:past + n].copy_(attention_mask[:, -n:] == 0)
        else:
            self.key_mask_known = False

    def reset(self):
        super().reset()
        self.key_mask_known = True
        self.eager_writes += 1

    def crop(self, max_length):
        super().crop(max_length)
        self.eager_writes += 1

    def reorder_cache(self, beam_idx):
        super().reorder_cache(beam_idx)
        if self.key_mask is not None and self.get_seq_length() > 0:
            self.key_mask.copy_(self.key_mask.index_select(0, beam_idx.to(self.key_mask.device)))
