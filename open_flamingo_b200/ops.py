"""Thin, shape-checked Python wrappers over the libofk.so C ABI (one function per entry point).

These do no math of their own.  Argument-shape violations raise ValueError/AssertionError *before* the
call (mirroring the reference's conventions, e.g. helpers.py:175-178); nonzero return codes from the
library become RuntimeError.
"""
import os

import torch

from . import _lib as L

bf16 = torch.bfloat16
f32 = torch.float32


def _rowmajor_2d(t, name):
    if t.dim() != 2 or t.stride(1) != 1:
        raise ValueError(f"{name} must be 2-D with unit inner stride, got shape {tuple(t.shape)} stride {t.stride()}")


def _vector(t, name, dtype, n, at_least=False):
    """t: a contiguous `dtype` tensor of exactly n elements (at least n with at_least)."""
    if t.dtype != dtype or not t.is_contiguous() or (t.numel() < n if at_least else t.numel() != n):
        raise ValueError(f"{name} must be a contiguous {dtype} tensor of {'>= ' if at_least else ''}{n} elements, got "
                         f"{tuple(t.shape)} {t.dtype} stride {t.stride()}")


def _rows2d(t, name, dtypes, rows, D):
    """t: 2-D, unit inner stride, one of `dtypes`, at least `rows` rows of at least D columns."""
    _rowmajor_2d(t, name)
    if t.dtype not in dtypes or t.shape[0] < rows or t.shape[1] < D:
        raise ValueError(f"{name} must be a {' or '.join(map(str, dtypes))} tensor of >= {rows} rows and >= {D} columns, "
                         f"got {tuple(t.shape)} {t.dtype}")


def _mapped_rows(rows, rows_per_group, group_stride, group_offset):
    """Rows of the buffer the LayerNorm group mapping reaches (row r -> (r // rpg) * stride + offset + r % rpg)."""
    if rows_per_group <= 0:
        return rows
    if group_offset < 0 or group_offset + rows_per_group > group_stride:
        raise ValueError(f"layernorm group mapping: need 0 <= group_offset and group_offset + rows_per_group <= "
                         f"group_stride, got ({rows_per_group}, {group_stride}, {group_offset})")
    last = rows - 1
    return (last // rows_per_group) * group_stride + group_offset + last % rows_per_group + 1


_comm_in_flight = False
# SMs every persistent GEMM grid leaves to NCCL while gradient-chunk all-reduces are in flight (world > 1 only; 0 = none).
# A persistent grid that owns every SM lets the all-reduce kernels in only at GEMM boundaries, so the "overlapped" reduction
# is serialised behind the GEMMs; 16 free SMs (with NCCL_MAX_CTAS=16, see train.configure_nccl_for_overlap) let it run
# beside them.  Not measured on H100 (the multi-GPU step needs more than one GPU).
COMM_RESERVED_SMS = int(os.environ.get("OFK_COMM_RESERVE_SMS", "16"))


def set_comm_in_flight(flag):
    """train.GradBucket brackets the window in which gradient-chunk all-reduces may be running.  Inside it the
    persistent GEMM grids are shrunk by COMM_RESERVED_SMS so the collective's CTAs can run BESIDE the GEMMs instead of
    between them."""
    global _comm_in_flight
    flag = bool(flag)
    if flag != _comm_in_flight and COMM_RESERVED_SMS > 0:
        L.lib().ofk_gemm_reserve_sms(COMM_RESERVED_SMS if flag else 0)
    _comm_in_flight = flag


def gemm(a, b, *, a_mn=False, b_mn=False, epi=L.EPI_STORE_BF16, out=None, out2=None, aux=None, bias=None,
         gate=None, splits=1, block_n=0, M=None, N=None, K=None):
    """out[m,n] = epi(sum_k A(m,k) B(n,k)).

    a: [M,K] (a_mn=False) or [K,M] (a_mn=True); b: [N,K] (b_mn=False) or [K,N] (b_mn=True); both bf16.
    """
    L.require_cuda(a, b)
    _rowmajor_2d(a, "a")
    _rowmajor_2d(b, "b")
    if a.dtype != bf16 or b.dtype != bf16:
        raise ValueError("gemm operands must be bfloat16")
    m, ka = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    n, kb = (b.shape[1], b.shape[0]) if b_mn else (b.shape[0], b.shape[1])
    if ka != kb:
        raise ValueError(f"gemm reduction dims differ: {ka} vs {kb}")
    M = m if M is None else M
    N = n if N is None else N
    K = ka if K is None else K
    out_dtype = f32 if epi in (L.EPI_STORE_F32, L.EPI_ATOMIC_F32, L.EPI_GATE_RESID_F32,
                               L.EPI_BIAS_RESID_F32) else bf16
    if out is None:
        if epi == L.EPI_ATOMIC_F32:
            raise ValueError("atomic epilogue accumulates into an existing `out`")
        out = torch.empty((M, N), device=a.device, dtype=out_dtype)
    _rowmajor_2d(out, "out")
    if out.dtype != out_dtype or out.shape[0] < M or out.shape[1] < N:
        raise ValueError(f"bad out tensor {tuple(out.shape)} {out.dtype} for ({M},{N}) {out_dtype}")
    if out2 is not None:
        _rowmajor_2d(out2, "out2")
        if out2.dtype != bf16 or out2.shape[0] < M or out2.shape[1] < N:
            raise ValueError(f"bad out2 tensor {tuple(out2.shape)} {out2.dtype} for ({M},{N}) {bf16}")
    if aux is not None:
        _rowmajor_2d(aux, "aux")
        aux_dtype = bf16 if epi == L.EPI_DGELU_BF16 else f32
        if epi in (L.EPI_GATE_RESID_F32, L.EPI_BIAS_RESID_F32, L.EPI_DGELU_BF16) and (
                aux.dtype != aux_dtype or aux.shape[0] < M or aux.shape[1] < N):
            raise ValueError(f"bad aux tensor {tuple(aux.shape)} {aux.dtype} for ({M},{N}) {aux_dtype}")
    if bias is not None and (bias.dtype != f32 or bias.numel() < N or not bias.is_contiguous()):
        raise ValueError("gemm bias must be a contiguous float32 vector of length >= N")
    if gate is not None and gate.dtype != f32:
        raise ValueError("gemm gate must be float32")
    L.check(L.lib().ofk_gemm_bf16(
        epi, int(a_mn), int(b_mn), a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), M, N, K, splits, block_n,
        out.data_ptr(), out.stride(0), L.ptr(out2), 0 if out2 is None else out2.stride(0),
        L.ptr(aux), 0 if aux is None else aux.stride(0), L.ptr(bias), L.ptr(gate), L.stream_ptr()))
    return out


def layernorm_fwd(x, gamma, beta, eps=1e-5, *, out=None, out_f32=False, rows_per_group=0, group_stride=0,
                  group_offset=0, want_stats=True):
    """x: [rows, D] f32.  Returns (y, mean, rstd).  `out` may be a larger buffer written with the group mapping."""
    L.require_cuda(x)
    _rowmajor_2d(x, "x")
    if x.dtype != f32:
        raise ValueError("layernorm input must be float32 (the residual stream is fp32)")
    rows, D = x.shape
    L.require_cuda(gamma, beta, out)
    _vector(gamma, "gamma", f32, D)
    _vector(beta, "beta", f32, D)
    if out is None:
        out = torch.empty((rows, D), device=x.device, dtype=f32 if out_f32 else bf16)
    _rows2d(out, "out", (f32, bf16), _mapped_rows(rows, rows_per_group, group_stride, group_offset), D)
    y_is_f32 = out.dtype == f32
    mean = torch.empty(rows, device=x.device, dtype=f32) if want_stats else None
    rstd = torch.empty(rows, device=x.device, dtype=f32) if want_stats else None
    L.check(L.lib().ofk_layernorm_fwd(x.data_ptr(), x.stride(0), gamma.data_ptr(), beta.data_ptr(), eps, rows, D,
                                      out.data_ptr(), int(y_is_f32), out.stride(0), rows_per_group, group_stride,
                                      group_offset, L.ptr(mean), L.ptr(rstd), L.stream_ptr()))
    return out, mean, rstd


_ln_ws = {}


def _ln_workspace(device, rows, D):
    need = int(L.lib().ofk_layernorm_bwd_workspace(rows, D))
    key = (device, torch.cuda.current_stream().cuda_stream)
    ws = _ln_ws.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, device=device, dtype=torch.uint8)
        _ln_ws[key] = ws
    return ws


def layernorm_bwd(dy, x, gamma, mean, rstd, *, dgamma=None, dbeta=None, dx=None, dx_add=None, rows_per_group=0,
                  group_stride=0, group_offset=0, want_dx=True):
    """dx = LN'(dy) (+ dx_add); dgamma/dbeta are accumulated in place.  dy may be bf16 or f32 (mapped rows).
    want_dx=False: only the affine-parameter gradients are produced."""
    L.require_cuda(dy, x, gamma, mean, rstd, dgamma, dbeta, dx, dx_add)
    _rowmajor_2d(x, "x")
    if x.dtype != f32:
        raise ValueError("layernorm input must be float32 (the residual stream is fp32)")
    rows, D = x.shape
    _rows2d(dy, "dy", (f32, bf16), _mapped_rows(rows, rows_per_group, group_stride, group_offset), D)
    _vector(gamma, "gamma", f32, D)
    _vector(mean, "mean", f32, rows)
    _vector(rstd, "rstd", f32, rows)
    for t, name in ((dgamma, "dgamma"), (dbeta, "dbeta")):
        if t is not None:
            _vector(t, name, f32, D)
    for t, name in ((dx, "dx"), (dx_add, "dx_add")):
        if t is not None:
            _rows2d(t, name, (f32,), rows, D)
    if dx is None and want_dx:
        dx = torch.empty((rows, D), device=x.device, dtype=f32)
    ws = _ln_workspace(x.device, rows, D)
    L.check(L.lib().ofk_layernorm_bwd(dy.data_ptr(), int(dy.dtype == f32), dy.stride(0), rows_per_group, group_stride,
                                      group_offset, x.data_ptr(), x.stride(0), gamma.data_ptr(), mean.data_ptr(),
                                      rstd.data_ptr(), rows, D, L.ptr(dx), 0 if dx is None else dx.stride(0), L.ptr(dx_add),
                                      0 if dx_add is None else dx_add.stride(0), L.ptr(dgamma), L.ptr(dbeta),
                                      ws.data_ptr(), L.stream_ptr()))
    return dx


def _bstride_ld(t, name):
    if t.dim() != 3 or t.stride(2) != 1:
        raise ValueError(f"{name} must be [batch, rows, heads*64] with unit inner stride")
    return t.stride(0), t.stride(1)


def _attn_qkv(q, k, v, inner):
    """Shape checks shared by the attention wrappers; returns (B, nq, nk)."""
    if q.dtype != bf16 or k.dtype != bf16 or v.dtype != bf16:
        raise ValueError("attention operands must be bfloat16")
    for t, name in ((q, "q"), (k, "k"), (v, "v")):
        if t.dim() != 3 or t.shape[2] != inner:
            raise ValueError(f"{name} must be [batch, rows, {inner}], got {tuple(t.shape)}")
    if tuple(k.shape) != tuple(v.shape) or k.shape[0] != q.shape[0]:
        raise ValueError(f"k {tuple(k.shape)} and v {tuple(v.shape)} must have the same shape and q's batch")
    return q.shape[0], q.shape[1], k.shape[1]


def _attn_rows(t, name, shape):
    """An o / d_o / dq / dk / dv tensor: bf16 with exactly the given [batch, rows, heads*head_dim] shape."""
    if t.dtype != bf16 or tuple(t.shape) != shape:
        raise ValueError(f"{name} must be a bf16 tensor of shape {shape}, got {tuple(t.shape)} {t.dtype}")


def _attn_lse(lse, B, heads, nq):
    if lse.dtype != f32 or tuple(lse.shape) != (B, heads, nq) or not lse.is_contiguous():
        raise ValueError(f"lse must be a contiguous float32 tensor of shape {(B, heads, nq)}")


def _attn_text_time(text_time, B, nq):
    if text_time is None or text_time.dtype != torch.int32 or tuple(text_time.shape) != (B, nq):
        raise ValueError("media mask needs int32 text_time of shape [B, nq]")
    return text_time.contiguous()


def _attn_strides(*named):
    """(batch stride, row stride) of each (tensor, name) pair, flattened in order."""
    return tuple(st for t, name in named for st in _bstride_ld(t, name))


def _attn_fwd_outputs(q, B, heads, nq, inner, out, want_lse):
    """o (allocated unless given) and lse (None unless wanted) of a forward call."""
    if out is None:
        out = torch.empty((B, nq, inner), device=q.device, dtype=bf16)
    _attn_rows(out, "out", (B, nq, inner))
    lse = torch.empty((B, heads, nq), device=q.device, dtype=f32) if want_lse else None
    return out, lse


def _attn_bwd_buffers(q, k, v, o, d_o, lse, heads, inner, dq, dk, dv):
    """Checks shared by the backward wrappers; allocates the gradients not given and delta.
    Returns (B, nq, nk, dq, dk, dv, delta)."""
    B, nq, nk = _attn_qkv(q, k, v, inner)
    _attn_rows(o, "o", (B, nq, inner))
    _attn_rows(d_o, "d_o", (B, nq, inner))
    if d_o.stride() != o.stride():
        raise ValueError("d_o must have the same strides as o")
    _attn_lse(lse, B, heads, nq)
    grads = []
    for t, name, n in ((dq, "dq", nq), (dk, "dk", nk), (dv, "dv", nk)):
        if t is None:
            t = torch.empty((B, n, inner), device=q.device, dtype=bf16)
        _attn_rows(t, name, (B, n, inner))
        grads.append(t)
    delta = torch.empty((B, heads, nq), device=q.device, dtype=f32)
    return (B, nq, nk, *grads, delta)


def _dense_mask_slopes(mask, slopes, pure_causal_flag, B, heads, nq, nk):
    # the kernel indexes mask as a contiguous [B, nq, nk] byte array and reads slopes[h]
    if mask is not None and (tuple(mask.shape) != (B, nq, nk) or not mask.is_contiguous() or mask.element_size() != 1):
        raise ValueError("mask must be a contiguous 1-byte tensor of shape [B, nq, nk]")
    if slopes is not None and (slopes.dtype != f32 or slopes.numel() < heads or not slopes.is_contiguous()):
        raise ValueError("slopes must be a contiguous float32 vector of length >= heads")
    if pure_causal_flag is not None and (pure_causal_flag.dtype != torch.int32 or pure_causal_flag.numel() < 1):
        raise ValueError("pure_causal_flag must be an int32 device tensor")


def attn_fwd(q, k, v, heads, scale, *, mask_mode=L.MASK_NONE, text_time=None, keys_per_media=64, out=None,
             want_lse=True):
    """q: [B, nq, heads*64] (may be a column-slice view), k/v: [B, nk, heads*64].  Returns (o, lse)."""
    L.require_cuda(q, k, v, out, text_time)
    B, nq, nk = _attn_qkv(q, k, v, heads * 64)
    out, lse = _attn_fwd_outputs(q, B, heads, nq, heads * 64, out, want_lse)
    strides = _attn_strides((q, "q"), (k, "k"), (v, "v"), (out, "out"))
    if mask_mode != L.MASK_NONE:
        text_time = _attn_text_time(text_time, B, nq)
    L.check(L.lib().ofk_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), L.ptr(lse), B, heads, nq, nk,
                                 *strides, scale, mask_mode, L.ptr(text_time), keys_per_media, L.stream_ptr()))
    return out, lse


def attn_bwd(q, k, v, o, d_o, lse, heads, scale, *, mask_mode=L.MASK_NONE, text_time=None, keys_per_media=64,
             dq=None, dk=None, dv=None):
    """Returns (dq, dk, dv) bf16.  d_o must share o's strides."""
    L.require_cuda(q, k, v, o, d_o, lse, dq, dk, dv, text_time)
    B, nq, nk, dq, dk, dv, delta = _attn_bwd_buffers(q, k, v, o, d_o, lse, heads, heads * 64, dq, dk, dv)
    if mask_mode != L.MASK_NONE:
        text_time = _attn_text_time(text_time, B, nq)
    strides = _attn_strides((q, "q"), (k, "k"), (v, "v"), (o, "o"), (dq, "dq"), (dk, "dk"), (dv, "dv"))
    L.check(L.lib().ofk_attn_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), d_o.data_ptr(), lse.data_ptr(),
                                 delta.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), B, heads, nq, nk,
                                 *strides, scale, mask_mode, L.ptr(text_time), keys_per_media, L.stream_ptr()))
    return dq, dk, dv


def make_labels(input_ids, pad_token_id, media_token_id, endofchunk_token_id=None, interleaved=False, out=None):
    """Device-side training labels (train_utils.py:102-106; interleaved=True: the MMC4 rule of :126-149).
    input_ids: int64 [B, T] on the GPU (row stride free).  Returns int64 [B, T]."""
    L.require_cuda(input_ids)
    if input_ids.dtype != torch.int64 or input_ids.dim() != 2 or (input_ids.numel() and input_ids.stride(1) != 1):
        raise ValueError("make_labels expects an int64 [B, T] tensor with contiguous rows")
    if interleaved and endofchunk_token_id is None:
        raise ValueError("interleaved labels need the <|endofchunk|> token id")
    B, T = input_ids.shape
    if out is None:
        out = torch.empty((B, T), device=input_ids.device, dtype=torch.int64)
    if B == 0 or T == 0:
        return out
    L.check(L.lib().ofk_make_labels(input_ids.data_ptr(), input_ids.stride(0), B, T, int(pad_token_id),
                                    int(media_token_id), int(-1 if endofchunk_token_id is None else endofchunk_token_id),
                                    int(bool(interleaved)), out.data_ptr(), out.stride(0), L.stream_ptr()))
    return out


def text_time(input_ids=None, media_token_id=0, media_locations=None, use_cached_media=False, t_txt=None):
    """int32 [B, T_txt] inclusive count of media tokens (helpers.py:199-208)."""
    src = media_locations if media_locations is not None else input_ids
    L.require_cuda(src)
    B = src.shape[0]
    n_loc = src.shape[1]
    if t_txt is None:
        t_txt = n_loc
    loc = None
    if media_locations is not None:
        loc = media_locations.to(torch.uint8).contiguous()
    ids = None
    if input_ids is not None and media_locations is None:
        ids = input_ids.to(torch.int64).contiguous()
    out = torch.empty((B, t_txt), device=src.device, dtype=torch.int32)
    L.check(L.lib().ofk_text_time(L.ptr(ids), int(media_token_id), B, t_txt, n_loc, L.ptr(loc), int(use_cached_media),
                                  out.data_ptr(), L.stream_ptr()))
    return out


def cast_bf16(src, out=None):
    L.require_cuda(src, out)
    if src.dtype != f32:
        raise ValueError("cast_bf16 source must be float32")
    src = src.contiguous()
    if out is None:
        out = torch.empty(src.shape, device=src.device, dtype=bf16)
    _vector(out, "out", bf16, src.numel())
    L.check(L.lib().ofk_cast_f32_bf16(src.data_ptr(), out.data_ptr(), src.numel(), L.stream_ptr()))
    return out


_reduce_ws = {}


def _reduce_workspace(device):
    """Per-block partials of the grid-wide sums (ofk_reduce_workspace_bytes), one buffer per (device, stream)."""
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    ws = _reduce_ws.get(key)
    if ws is None:
        ws = torch.empty(int(L.lib().ofk_reduce_workspace_bytes()) // 4, device=device, dtype=f32)
        _reduce_ws[key] = ws
    return ws


def gate_bwd(dout, branch, gate, dgate):
    """dbranch(bf16) = dout * tanh(gate); dgate += (1 - tanh^2) * <dout, branch>.  gate None: plain cast."""
    L.require_cuda(dout, branch, gate, dgate)
    _vector(dout, "dout", f32, dout.numel())
    if gate is not None:
        _vector(gate, "gate", f32, 1)
        if branch is None:
            raise ValueError("gate_bwd with a gate needs the branch")
        _vector(branch, "branch", bf16, dout.numel())
    if dgate is not None:
        _vector(dgate, "dgate", f32, 1)
    dbranch = torch.empty(dout.shape, device=dout.device, dtype=bf16)
    ws = _reduce_workspace(dout.device) if (gate is not None and dgate is not None) else None
    L.check(L.lib().ofk_gate_bwd(dout.data_ptr(), L.ptr(branch), L.ptr(gate), dbranch.data_ptr(), L.ptr(dgate),
                                 dout.numel(), L.ptr(ws), L.stream_ptr()))
    return dbranch


def add_(dst, src):
    """dst += src, both contiguous float32 of the same size."""
    L.require_cuda(dst, src)
    _vector(dst, "dst", f32, dst.numel())
    _vector(src, "src", f32, dst.numel())
    L.check(L.lib().ofk_add_f32(dst.data_ptr(), src.data_ptr(), dst.numel(), L.stream_ptr()))
    return dst


def patchify(images, patch, ldp):
    """images [n,3,H,W] f32 -> [n*g, ldp] bf16 patch rows (conv-weight column order), zero padded."""
    L.require_cuda(images)
    if images.dtype != f32 or images.dim() != 4 or images.shape[1] != 3:
        raise ValueError(f"images must be float32 [n, 3, H, W], got {tuple(images.shape)} {images.dtype}")
    images = images.contiguous()
    n, _, H, W = images.shape
    g = (H // patch) * (W // patch)
    out = torch.empty((n * g, ldp), device=images.device, dtype=bf16)
    L.check(L.lib().ofk_patchify(images.data_ptr(), n, H, W, patch, out.data_ptr(), ldp, L.stream_ptr()))
    return out


def vit_assemble(patch_emb, class_emb, pos_emb, n, g, D):
    """patch_emb: contiguous bf16 [n*g, D]; class_emb: f32 [D]; pos_emb: contiguous f32 [g+1, D].  Returns f32
    [n*(g+1), D] tokens."""
    L.require_cuda(patch_emb, class_emb, pos_emb)
    if patch_emb.dtype != bf16 or tuple(patch_emb.shape) != (n * g, D) or not patch_emb.is_contiguous():
        raise ValueError(f"patch_emb must be a contiguous bf16 [{n * g}, {D}] tensor, got {tuple(patch_emb.shape)} "
                         f"{patch_emb.dtype}")
    _vector(class_emb, "class_emb", f32, D)
    if pos_emb.dtype != f32 or tuple(pos_emb.shape) != (g + 1, D) or not pos_emb.is_contiguous():
        raise ValueError(f"pos_emb must be a contiguous float32 [{g + 1}, {D}] tensor, got {tuple(pos_emb.shape)} "
                         f"{pos_emb.dtype}")
    tok = torch.empty((n * (g + 1), D), device=patch_emb.device, dtype=f32)
    L.check(L.lib().ofk_vit_assemble(patch_emb.data_ptr(), class_emb.data_ptr(), pos_emb.data_ptr(), n, g, D,
                                     tok.data_ptr(), L.stream_ptr()))
    return tok


def adamw_(param, grad, exp_avg, exp_avg_sq, w_bf16, lr, beta1, beta2, eps, wd, step, clip_scale=None, step_dev=None,
           lr_dev=None):
    """step: host int (ignored when step_dev, a device float tensor holding the step count, is given).
    param, grad, exp_avg, exp_avg_sq: contiguous float32 of one size; w_bf16: contiguous bf16 of that size or None;
    clip_scale, step_dev, lr_dev: float32 device scalars or None."""
    L.require_cuda(param, grad, exp_avg, exp_avg_sq, w_bf16, clip_scale, step_dev, lr_dev)
    n = param.numel()
    for t, name in ((param, "param"), (grad, "grad"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        _vector(t, name, f32, n)
    if w_bf16 is not None:
        _vector(w_bf16, "w_bf16", bf16, n)
    for t, name in ((clip_scale, "clip_scale"), (step_dev, "step_dev"), (lr_dev, "lr_dev")):
        if t is not None:
            _vector(t, name, f32, 1, at_least=True)
    bc1 = 1.0 - beta1 ** max(step, 1)
    bc2 = 1.0 - beta2 ** max(step, 1)
    L.check(L.lib().ofk_adamw(param.data_ptr(), grad.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(),
                              L.ptr(w_bf16), param.numel(), lr, beta1, beta2, eps, wd, bc1, bc2, L.ptr(clip_scale),
                              L.ptr(step_dev), L.ptr(lr_dev), L.stream_ptr()))


def sumsq_(x, out):
    """out[0] += sum(x * x); x contiguous float32, out a float32 device scalar."""
    L.require_cuda(x, out)
    _vector(x, "x", f32, x.numel())
    _vector(out, "out", f32, 1, at_least=True)
    L.check(L.lib().ofk_sumsq(x.data_ptr(), x.numel(), out.data_ptr(), _reduce_workspace(x.device).data_ptr(),
                              L.stream_ptr()))
    return out


def attn_dense_fwd(q, k, v, heads, head_dim, scale, *, causal=False, mask=None, slopes=None, pure_causal_flag=None,
                   want_lse=True):
    """Dense (LM self-attention) core: q/k/v [B, n, heads*head_dim] strided views; mask [B, nq, nk] bool/uint8
    (True = masked); slopes [heads] f32 ALiBi slopes.  Returns (o, lse)."""
    L.require_cuda(q, k, v, mask, slopes, pure_causal_flag)
    B, nq, nk = _attn_qkv(q, k, v, heads * head_dim)
    _dense_mask_slopes(mask, slopes, pure_causal_flag, B, heads, nq, nk)
    out, lse = _attn_fwd_outputs(q, B, heads, nq, heads * head_dim, None, want_lse)
    strides = _attn_strides((q, "q"), (k, "k"), (v, "v"), (out, "out"))
    L.check(L.lib().ofk_attn_dense_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), L.ptr(lse), B, heads,
                                       head_dim, nq, nk, *strides, scale, int(causal), L.ptr(mask), L.ptr(slopes),
                                       L.ptr(pure_causal_flag), L.stream_ptr()))
    return out, lse


_decode_ws = {}


def _decode_workspace(device, B, heads, head_dim, nk):
    """Split partials of ofk_attn_decode, one grow-only buffer per (device, stream)."""
    need = int(L.lib().ofk_attn_decode_workspace_bytes(B, heads, head_dim, nk))
    if need < 0:
        raise ValueError(f"attn_decode: unsupported problem (batch {B}, heads {heads}, head_dim {head_dim}, nk {nk})")
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    ws = _decode_ws.get(key)
    if ws is None or ws.numel() * 4 < need:
        ws = torch.empty((need + 3) // 4, device=device, dtype=f32)
        _decode_ws[key] = ws
    return ws


def attn_decode(q, k, v, heads, head_dim, scale, *, key_mask=None, slopes=None, out=None):
    """Decode attention (one query row per batch entry and head) over the first nk rows of a K/V cache.
    q: [B, heads*head_dim] with unit inner stride (e.g. a column slice of a qkv row); k/v: [B, nk, heads*head_dim] views
    with the same strides (the K and V column slices of one cache buffer); key_mask: [B, >= nk] 1-byte tensor
    (nonzero = masked) with unit inner stride; slopes: [heads] f32 ALiBi slopes.  Returns o [B, heads*head_dim] bf16."""
    L.require_cuda(q, k, v, key_mask, slopes)
    if q.dtype != bf16 or k.dtype != bf16 or v.dtype != bf16:
        raise ValueError("attention operands must be bfloat16")
    inner = heads * head_dim
    if q.dim() != 2 or q.shape[1] != inner or q.stride(1) != 1:
        raise ValueError(f"q must be [B, {inner}] with unit inner stride, got {tuple(q.shape)} stride {q.stride()}")
    B = q.shape[0]
    if k.dim() != 3 or tuple(k.shape) != tuple(v.shape) or k.shape[0] != B or k.shape[2] != inner or \
            k.stride(2) != 1 or k.stride() != v.stride():
        raise ValueError(f"k/v must be [B, nk, {inner}] views with equal strides and unit inner stride, got "
                         f"{tuple(k.shape)} {k.stride()} / {tuple(v.shape)} {v.stride()}")
    nk = k.shape[1]
    if key_mask is not None and (key_mask.dim() != 2 or key_mask.shape[0] != B or key_mask.shape[1] < nk or
                                 key_mask.element_size() != 1 or key_mask.stride(1) != 1):
        raise ValueError(f"key_mask must be a 1-byte [B, >= {nk}] tensor with unit inner stride")
    if slopes is not None and (slopes.dtype != f32 or slopes.numel() < heads or not slopes.is_contiguous()):
        raise ValueError("slopes must be a contiguous float32 vector of length >= heads")
    if out is None:
        out = torch.empty((B, inner), device=q.device, dtype=bf16)
    elif out.dtype != bf16 or out.dim() != 2 or tuple(out.shape) != (B, inner) or out.stride(1) != 1:
        raise ValueError(f"out must be a bf16 [B, {inner}] tensor with unit inner stride")
    ws = _decode_workspace(q.device, B, heads, head_dim, nk)
    L.check(L.lib().ofk_attn_decode(q.data_ptr(), q.stride(0), k.data_ptr(), v.data_ptr(), k.stride(0), k.stride(1),
                                    out.data_ptr(), out.stride(0), B, heads, head_dim, nk, scale, L.ptr(key_mask),
                                    0 if key_mask is None else key_mask.stride(0), L.ptr(slopes), ws.data_ptr(),
                                    L.stream_ptr()))
    return out


def decode_workspace(device, B, heads, head_dim, nk_max):
    """A workspace of its own for attn_decode_dev: a captured graph keeps using the buffer it was captured with, so it
    must not come from the grow-only per-stream buffers that eager calls may replace."""
    need = int(L.lib().ofk_attn_decode_workspace_bytes(B, heads, head_dim, nk_max))
    if need < 0:
        raise ValueError(f"attn_decode: unsupported problem (batch {B}, heads {heads}, head_dim {head_dim}, "
                         f"nk_max {nk_max})")
    return torch.empty((need + 3) // 4, device=device, dtype=f32)


def attn_decode_dev(q, k, v, heads, head_dim, scale, nk_dev, *, key_mask=None, slopes=None, out=None, workspace=None):
    """attn_decode with the key count read on the device: nk = min(nk_dev[0], nk_max), nk_max = k.shape[1] (the cache's
    capacity).  Bitwise equal to attn_decode over the first nk rows.  nk_dev: int32 CUDA tensor; workspace: a float32
    tensor of at least ofk_attn_decode_workspace_bytes(B, heads, head_dim, nk_max) bytes (see decode_workspace)."""
    L.require_cuda(q, k, v, key_mask, slopes, nk_dev, workspace)
    if q.dtype != bf16 or k.dtype != bf16 or v.dtype != bf16:
        raise ValueError("attention operands must be bfloat16")
    inner = heads * head_dim
    if q.dim() != 2 or q.shape[1] != inner or q.stride(1) != 1:
        raise ValueError(f"q must be [B, {inner}] with unit inner stride, got {tuple(q.shape)} stride {q.stride()}")
    B = q.shape[0]
    if k.dim() != 3 or tuple(k.shape) != tuple(v.shape) or k.shape[0] != B or k.shape[2] != inner or \
            k.stride(2) != 1 or k.stride() != v.stride():
        raise ValueError(f"k/v must be [B, nk_max, {inner}] views with equal strides and unit inner stride, got "
                         f"{tuple(k.shape)} {k.stride()} / {tuple(v.shape)} {v.stride()}")
    nk_max = k.shape[1]
    if key_mask is not None and (key_mask.dim() != 2 or key_mask.shape[0] != B or key_mask.shape[1] < nk_max or
                                 key_mask.element_size() != 1 or key_mask.stride(1) != 1):
        raise ValueError(f"key_mask must be a 1-byte [B, >= {nk_max}] tensor with unit inner stride")
    if slopes is not None and (slopes.dtype != f32 or slopes.numel() < heads or not slopes.is_contiguous()):
        raise ValueError("slopes must be a contiguous float32 vector of length >= heads")
    if nk_dev.dtype != torch.int32 or nk_dev.numel() < 1:
        raise ValueError("nk_dev must be an int32 device tensor")
    if out is None:
        out = torch.empty((B, inner), device=q.device, dtype=bf16)
    elif out.dtype != bf16 or out.dim() != 2 or tuple(out.shape) != (B, inner) or out.stride(1) != 1:
        raise ValueError(f"out must be a bf16 [B, {inner}] tensor with unit inner stride")
    if workspace is None:
        workspace = decode_workspace(q.device, B, heads, head_dim, nk_max)
    elif workspace.numel() * workspace.element_size() < int(L.lib().ofk_attn_decode_workspace_bytes(
            B, heads, head_dim, nk_max)):
        raise ValueError("attn_decode_dev: workspace too small for nk_max")
    L.check(L.lib().ofk_attn_decode_dev(q.data_ptr(), q.stride(0), k.data_ptr(), v.data_ptr(), k.stride(0), k.stride(1),
                                        out.data_ptr(), out.stride(0), B, heads, head_dim, nk_max, nk_dev.data_ptr(),
                                        scale, L.ptr(key_mask), 0 if key_mask is None else key_mask.stride(0),
                                        L.ptr(slopes), workspace.data_ptr(), L.stream_ptr()))
    return out


def kv_append(src, cache, pos_dev, *, key_mask=None, new_masked=None):
    """cache[b, pos, :] = src[b, :] at the device-side position pos = pos_dev[0] (nothing outside [0, capacity)), and
    key_mask[b, pos] = new_masked[b] != 0 (0 when new_masked is None).  src: [B, W] bf16 with unit inner stride;
    cache: [B, capacity, W] bf16 view with unit inner stride; key_mask: 1-byte [B, >= capacity] with unit inner stride;
    new_masked: 1-byte [B]; pos_dev: int32 CUDA tensor."""
    L.require_cuda(src, cache, pos_dev, key_mask, new_masked)
    if src.dtype != bf16 or cache.dtype != bf16:
        raise ValueError("kv_append operands must be bfloat16")
    if src.dim() != 2 or src.stride(1) != 1:
        raise ValueError(f"src must be [B, W] with unit inner stride, got {tuple(src.shape)} stride {src.stride()}")
    B, W = src.shape
    if cache.dim() != 3 or cache.shape[0] != B or cache.shape[2] != W or cache.stride(2) != 1:
        raise ValueError(f"cache must be a [{B}, capacity, {W}] view with unit inner stride, got {tuple(cache.shape)}")
    cap = cache.shape[1]
    if key_mask is not None and (key_mask.dim() != 2 or key_mask.shape[0] != B or key_mask.shape[1] < cap or
                                 key_mask.element_size() != 1 or key_mask.stride(1) != 1):
        raise ValueError(f"key_mask must be a 1-byte [B, >= {cap}] tensor with unit inner stride")
    if new_masked is not None and (new_masked.numel() != B or new_masked.element_size() != 1 or
                                   not new_masked.is_contiguous()):
        raise ValueError(f"new_masked must be a contiguous 1-byte tensor of {B} elements")
    if pos_dev.dtype != torch.int32 or pos_dev.numel() < 1:
        raise ValueError("pos_dev must be an int32 device tensor")
    L.check(L.lib().ofk_kv_append(src.data_ptr(), src.stride(0), cache.data_ptr(), cache.stride(0), cache.stride(1), B,
                                  W, cap, pos_dev.data_ptr(), L.ptr(key_mask),
                                  0 if key_mask is None else key_mask.stride(0), L.ptr(new_masked), L.stream_ptr()))
    return cache


def attn_dense_bwd(q, k, v, o, d_o, lse, heads, head_dim, scale, *, causal=False, mask=None, slopes=None,
                   pure_causal_flag=None, dq=None, dk=None, dv=None):
    L.require_cuda(q, k, v, o, d_o, lse, mask, slopes, pure_causal_flag, dq, dk, dv)
    B, nq, nk, dq, dk, dv, delta = _attn_bwd_buffers(q, k, v, o, d_o, lse, heads, heads * head_dim, dq, dk, dv)
    _dense_mask_slopes(mask, slopes, pure_causal_flag, B, heads, nq, nk)
    strides = _attn_strides((q, "q"), (k, "k"), (v, "v"), (o, "o"), (dq, "dq"), (dk, "dk"), (dv, "dv"))
    L.check(L.lib().ofk_attn_dense_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), d_o.data_ptr(),
                                       lse.data_ptr(), delta.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(),
                                       B, heads, head_dim, nq, nk, *strides, scale, int(causal), L.ptr(mask),
                                       L.ptr(slopes), L.ptr(pure_causal_flag), L.stream_ptr()))
    return dq, dk, dv


def gemm_grouped(a, b, *, a_mn=False, b_mn=False, epi=L.EPI_STORE_BF16, out, M, N, K, bias=None, splits=1, block_n=0,
                 out_map=(0, 0, 0), ak_map=(0, 0, 0)):
    """GEMM with grouped row maps (see ofk_gemm_bf16_grouped): `out_map` = (rows_per_group, group_stride,
    group_offset) for the rows of `out`, with M a whole number of groups; `ak_map` the same for the reduction rows of
    an MN-major `a`."""
    L.require_cuda(a, b, out)
    _rowmajor_2d(a, "a")
    _rowmajor_2d(b, "b")
    _rowmajor_2d(out, "out")
    if a.dtype != bf16 or b.dtype != bf16:
        raise ValueError("gemm operands must be bfloat16")
    if bias is not None and (bias.dtype != f32 or bias.numel() < N or not bias.is_contiguous()):
        raise ValueError("gemm bias must be a contiguous float32 vector of length >= N")
    L.check(L.lib().ofk_gemm_bf16_grouped(
        epi, int(a_mn), int(b_mn), a.data_ptr(), a.stride(0), b.data_ptr(), b.stride(0), M, N, K, splits, block_n,
        out.data_ptr(), out.stride(0), L.ptr(bias), out_map[0], out_map[1], out_map[2], ak_map[0], ak_map[1], ak_map[2],
        L.stream_ptr()))
    return out


def _rope_tables(cos, sin, B, rows, rot):
    """(cs_bstride, ld_cs) of fp32 cos/sin tables [1 or B, rows, rot] with unit inner stride and equal strides."""
    for t, name in ((cos, "cos"), (sin, "sin")):
        if t.dtype != f32 or t.dim() != 3 or t.shape[0] not in (1, B) or t.shape[1] != rows or t.shape[2] != rot or \
                t.stride(2) != 1:
            raise ValueError(f"{name} must be float32 [1 or {B}, {rows}, {rot}] with unit inner stride, got "
                             f"{tuple(t.shape)} {t.dtype} stride {t.stride()}")
    if cos.shape != sin.shape or cos.stride() != sin.stride():
        raise ValueError("cos and sin must have the same shape and strides")
    return (cos.stride(0) if cos.shape[0] == B and B > 1 else 0), cos.stride(1)


def _rope_dest(t, name, B, rows, inner):
    if t.dtype != bf16 or t.dim() != 3 or tuple(t.shape) != (B, rows, inner) or t.stride(2) != 1:
        raise ValueError(f"{name} must be a bf16 [{B}, {rows}, {inner}] view with unit inner stride, got "
                         f"{tuple(t.shape)} {t.dtype} stride {t.stride()}")
    return t.stride(0), t.stride(1)


def rope_pack(src, heads, head_dim, cos=None, sin=None, *, q=None, k=None, v=None, q_width=None, kv_width=None,
              kv_src=None, blocks=False):
    """Rotary q/k packing of GPT-NeoX rows (ofk_rope_pack).

    src: [B, T, heads * 3 * head_dim] bf16 view of the query_key_value output (heads interleaved as (q | k | v)), or
    None with kv_src = (k_rows, v_rows): two [B, T, heads * head_dim] views (the K and V columns of a KV cache) whose
    heads are only re-laid out.  blocks=True: src holds q, k and v as three column blocks of heads * head_dim each
    (nn.MultiheadAttention's in_proj output, as in the CLIP ViT).  cos/sin: fp32 [1 or B, T, rot] (None: no rotation).
    q / k / v: destinations [B, T, heads * width] (allocated when None and wanted); q_width, kv_width: head widths
    (default head_dim), columns past head_dim are zero.  Returns (q, k, v); q is None with kv_src."""
    L.require_cuda(src, cos, sin, q, k, v, *(kv_src or ()))
    q_width = head_dim if q_width is None else q_width
    kv_width = head_dim if kv_width is None else kv_width
    if src is not None:
        if src.dtype != bf16 or src.dim() != 3 or src.shape[2] != heads * 3 * head_dim or src.stride(2) != 1:
            raise ValueError(f"src must be a bf16 [B, T, {heads * 3 * head_dim}] view with unit inner stride, got "
                             f"{tuple(src.shape)} {src.dtype}")
        B, T = src.shape[:2]
        part = heads * head_dim if blocks else head_dim   # column offset of k's (and v's) head 0 after q's
        srcs = (src, src[..., part:], src[..., 2 * part:])
        sbs, sld, shs = src.stride(0), src.stride(1), head_dim if blocks else 3 * head_dim
    else:
        if blocks:
            raise ValueError("rope_pack: blocks=True describes src; it does not apply to kv_src")
        ks, vs = kv_src
        if ks.dtype != bf16 or ks.dim() != 3 or ks.shape != vs.shape or ks.stride() != vs.stride() or \
                ks.shape[2] != heads * head_dim or ks.stride(2) != 1:
            raise ValueError(f"kv_src must be two bf16 [B, T, {heads * head_dim}] views with equal strides")
        B, T = ks.shape[:2]
        srcs = (None, ks, vs)
        sbs, sld, shs = ks.stride(0), ks.stride(1), head_dim
    rot = 0
    cs_bs = ld_cs = 0
    if cos is not None:
        rot = cos.shape[-1]
        cs_bs, ld_cs = _rope_tables(cos, sin, B, T, rot)
    outs = []
    for t, name, w, s in ((q, "q", q_width, srcs[0]), (k, "k", kv_width, srcs[1]), (v, "v", kv_width, srcs[2])):
        if s is None:
            outs.append((None, 0, 0, 0))
            continue
        if t is None:
            t = torch.empty((B, T, heads * w), device=s.device, dtype=bf16)
        outs.append((t,) + _rope_dest(t, name, B, T, heads * w) + (w,))
    args = []
    for t, bs, ld, w in outs:
        args += [L.ptr(t), bs, ld, w]
    L.check(L.lib().ofk_rope_pack(L.ptr(srcs[0]), L.ptr(srcs[1]), L.ptr(srcs[2]), sbs, sld, shs, B, T, heads, head_dim,
                                  rot, L.ptr(cos), L.ptr(sin), cs_bs, ld_cs, *args, L.stream_ptr()))
    return outs[0][0], outs[1][0], outs[2][0]


def rope_append_dev(qkv, heads, head_dim, cos, sin, cache, pos_dev, *, key_mask=None, new_masked=None, q=None):
    """The one-token rope_pack of a captured decode step (ofk_rope_append_dev): rotates q and k of the interleaved
    query_key_value rows qkv [B, heads * 3 * head_dim] (bf16, unit inner stride) with cos/sin fp32 [1 or B, 1, rot]
    (None: no rotation), writes q to `q` [B, heads * head_dim] (allocated when None) and the rotated K and the V into
    row pos = pos_dev[0] of `cache` [B, capacity, 2 * heads * head_dim] (K columns, then V), and sets
    key_mask[b, pos] = new_masked[b] != 0 as kv_append does.  Nothing but q is written for a pos outside
    [0, capacity).  key_mask: 1-byte [B, >= capacity], unit inner stride; new_masked: 1-byte [B]; pos_dev: int32 CUDA
    tensor.  Returns q."""
    L.require_cuda(qkv, cos, sin, cache, pos_dev, key_mask, new_masked, q)
    D = heads * head_dim
    if qkv.dtype != bf16 or qkv.dim() != 2 or qkv.shape[1] != 3 * D or qkv.stride(1) != 1:
        raise ValueError(f"qkv must be a bf16 [B, {3 * D}] view with unit inner stride, got {tuple(qkv.shape)} "
                         f"{qkv.dtype}")
    B = qkv.shape[0]
    if cache.dtype != bf16 or cache.dim() != 3 or cache.shape[0] != B or cache.shape[2] != 2 * D or \
            cache.stride(2) != 1:
        raise ValueError(f"cache must be a bf16 [{B}, capacity, {2 * D}] view with unit inner stride, got "
                         f"{tuple(cache.shape)} {cache.dtype}")
    cap = cache.shape[1]
    rot = cs_bs = 0
    if cos is not None:
        rot = cos.shape[-1]
        cs_bs, _ = _rope_tables(cos, sin, B, 1, rot)
    if key_mask is not None and (key_mask.dim() != 2 or key_mask.shape[0] != B or key_mask.shape[1] < cap or
                                 key_mask.element_size() != 1 or key_mask.stride(1) != 1):
        raise ValueError(f"key_mask must be a 1-byte [B, >= {cap}] tensor with unit inner stride")
    if new_masked is not None and (new_masked.numel() != B or new_masked.element_size() != 1 or
                                   not new_masked.is_contiguous()):
        raise ValueError(f"new_masked must be a contiguous 1-byte tensor of {B} elements")
    if pos_dev.dtype != torch.int32 or pos_dev.numel() < 1:
        raise ValueError("pos_dev must be an int32 device tensor")
    if q is None:
        q = torch.empty((B, D), device=qkv.device, dtype=bf16)
    elif q.dtype != bf16 or q.dim() != 2 or tuple(q.shape) != (B, D) or q.stride(1) != 1:
        raise ValueError(f"q must be a bf16 [{B}, {D}] tensor with unit inner stride")
    L.check(L.lib().ofk_rope_append_dev(qkv.data_ptr(), qkv.stride(0), B, heads, head_dim, rot, L.ptr(cos), L.ptr(sin),
                                        cs_bs, q.data_ptr(), q.stride(0), cache.data_ptr(), cache.stride(0),
                                        cache.stride(1), cap, pos_dev.data_ptr(), L.ptr(key_mask),
                                        0 if key_mask is None else key_mask.stride(0), L.ptr(new_masked),
                                        L.stream_ptr()))
    return q


def rope_unpack_bwd(dq, dk, dv, heads, head_dim, cos=None, sin=None, *, out=None):
    """Adjoint of rope_pack (ofk_rope_unpack_bwd): dq/dk/dv [B, T, heads * W] bf16 views -> the gradient of the
    interleaved rows, [B, T, heads * 3 * head_dim] bf16 (`out`, allocated when None)."""
    L.require_cuda(dq, dk, dv, cos, sin, out)
    if dq.dim() != 3 or dq.shape[2] % heads != 0:
        raise ValueError(f"dq must be [B, T, heads * width], got {tuple(dq.shape)}")
    B, T, inner = dq.shape
    W = inner // heads
    strides = []
    for t, name in ((dq, "dq"), (dk, "dk"), (dv, "dv")):
        strides += list(_rope_dest(t, name, B, T, inner))
    rot = 0
    cs_bs = ld_cs = 0
    if cos is not None:
        rot = cos.shape[-1]
        cs_bs, ld_cs = _rope_tables(cos, sin, B, T, rot)
    if out is None:
        out = torch.empty((B, T, heads * 3 * head_dim), device=dq.device, dtype=bf16)
    obs, old = _rope_dest(out, "out", B, T, heads * 3 * head_dim)
    L.check(L.lib().ofk_rope_unpack_bwd(dq.data_ptr(), strides[0], strides[1], dk.data_ptr(), strides[2], strides[3],
                                        dv.data_ptr(), strides[4], strides[5], W, B, T, heads, head_dim, rot,
                                        L.ptr(cos), L.ptr(sin), cs_bs, ld_cs, out.data_ptr(), obs, old,
                                        L.stream_ptr()))
    return out


def gelu_bf16(z, out=None):
    """h = bf16(gelu_erf(z)) for a contiguous bf16 z, bit for bit the BIAS_GELU_BF16 epilogue's GELU."""
    L.require_cuda(z, out)
    _vector(z, "z", bf16, z.numel())
    if out is None:
        out = torch.empty(z.shape, device=z.device, dtype=bf16)
    _vector(out, "out", bf16, z.numel())
    L.check(L.lib().ofk_gelu_bf16(z.data_ptr(), out.data_ptr(), z.numel(), L.stream_ptr()))
    return out


def rmsnorm_fwd(x, gamma, eps, *, out=None, want_rstd=True):
    """RMSNorm (ofk_rmsnorm_fwd): x [rows, D] f32 with unit inner stride -> (y, rstd): y = bf16(gamma * (x * rstd))
    [rows, D] (`out`, allocated when None), rstd [rows] f32 (None unless want_rstd)."""
    L.require_cuda(x, gamma, out)
    _rowmajor_2d(x, "x")
    if x.dtype != f32:
        raise ValueError("rmsnorm input must be float32 (the residual stream is fp32)")
    rows, D = x.shape
    _vector(gamma, "gamma", f32, D)
    if out is None:
        out = torch.empty((rows, D), device=x.device, dtype=bf16)
    _rows2d(out, "out", (bf16,), rows, D)
    rstd = torch.empty(rows, device=x.device, dtype=f32) if want_rstd else None
    if rows:
        L.check(L.lib().ofk_rmsnorm_fwd(x.data_ptr(), x.stride(0), gamma.data_ptr(), float(eps), rows, D,
                                        out.data_ptr(), out.stride(0), L.ptr(rstd), L.stream_ptr()))
    return out, rstd


def rmsnorm_bwd(dy, x, gamma, rstd, *, dx=None, dx_add=None):
    """Input gradient of rmsnorm_fwd (ofk_rmsnorm_bwd): dy [rows, D] bf16 -> dx [rows, D] f32 (`dx`, allocated when
    None) = rstd * (gamma * dy - xhat * mean(gamma * dy * xhat)) + dx_add; dx_add may be dx itself."""
    L.require_cuda(dy, x, gamma, rstd, dx, dx_add)
    _rowmajor_2d(x, "x")
    if x.dtype != f32:
        raise ValueError("rmsnorm input must be float32 (the residual stream is fp32)")
    rows, D = x.shape
    _rows2d(dy, "dy", (bf16,), rows, D)
    _vector(gamma, "gamma", f32, D)
    _vector(rstd, "rstd", f32, rows)
    for t, name in ((dx, "dx"), (dx_add, "dx_add")):
        if t is not None:
            _rows2d(t, name, (f32,), rows, D)
    if dx is None:
        dx = torch.empty((rows, D), device=x.device, dtype=f32)
    if rows:
        L.check(L.lib().ofk_rmsnorm_bwd(dy.data_ptr(), dy.stride(0), x.data_ptr(), x.stride(0), gamma.data_ptr(),
                                        rstd.data_ptr(), rows, D, dx.data_ptr(), dx.stride(0), L.ptr(dx_add),
                                        0 if dx_add is None else dx_add.stride(0), L.stream_ptr()))
    return dx


def _swiglu_gu(gu):
    _rowmajor_2d(gu, "gu")
    if gu.dtype != bf16 or gu.shape[1] % 2:
        raise ValueError(f"gu must be bf16 [rows, 2F], got {tuple(gu.shape)} {gu.dtype}")
    return gu.shape[0], gu.shape[1] // 2


def swiglu_fwd(gu, out=None):
    """SwiGLU (ofk_swiglu_fwd): gu = [g | u] bf16 [rows, 2F] -> h = bf16(bf16(silu(g)) * u) [rows, F] (`out`,
    allocated when None)."""
    L.require_cuda(gu, out)
    rows, F = _swiglu_gu(gu)
    if out is None:
        out = torch.empty((rows, F), device=gu.device, dtype=bf16)
    _rows2d(out, "out", (bf16,), rows, F)
    if rows:
        L.check(L.lib().ofk_swiglu_fwd(gu.data_ptr(), gu.stride(0), rows, F, out.data_ptr(), out.stride(0),
                                       L.stream_ptr()))
    return out


def swiglu_bwd(dh, gu, out=None):
    """Gradient of swiglu_fwd (ofk_swiglu_bwd): dh bf16 [rows, F] -> dgu bf16 [rows, 2F] (`out`, allocated when
    None): [bf16(dh * u * silu'(g)) | bf16(dh * bf16(silu(g)))]."""
    L.require_cuda(dh, gu, out)
    rows, F = _swiglu_gu(gu)
    _rows2d(dh, "dh", (bf16,), rows, F)
    if out is None:
        out = torch.empty((rows, 2 * F), device=gu.device, dtype=bf16)
    _rows2d(out, "out", (bf16,), rows, 2 * F)
    if rows:
        L.check(L.lib().ofk_swiglu_bwd(dh.data_ptr(), dh.stride(0), gu.data_ptr(), gu.stride(0), rows, F,
                                       out.data_ptr(), out.stride(0), L.stream_ptr()))
    return out


def clip_preprocess(images, size, mean, std, *, out=None):
    """open_clip's eval transform (Resize(size, BICUBIC) + CenterCrop(size) + ToTensor + Normalize(mean, std)) of
    decoded images on the GPU, bit for bit torchvision + Pillow (ofk_image_plan + ofk_clip_preprocess: two launches for
    the whole batch).  images: a non-empty list of uint8 CUDA tensors [h, w, c], c = 1 (L) or 3 (RGB), channels and
    pixels contiguous, rows at any stride >= w * c.  Returns out: f32 [N, 3, size, size] (`out`, allocated when None;
    each image contiguous, images at any stride >= 3 size^2, so it may be a window of a larger vision_x buffer)."""
    import ctypes
    if not isinstance(images, (list, tuple)) or not images:
        raise ValueError("clip_preprocess needs a non-empty list of images")
    L.require_cuda(*images, out)
    S = int(size)
    if not 1 <= S <= 4096:
        raise ValueError(f"size must be in [1, 4096], got {size}")
    if len(mean) != 3 or len(std) != 3:
        raise ValueError("mean and std must have 3 entries")
    shape = []
    for i, t in enumerate(images):
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] not in (1, 3) or t.shape[0] < 1 or t.shape[1] < 1:
            raise ValueError(f"image {i} must be a uint8 [h, w, 1 or 3] tensor, got {tuple(t.shape)} {t.dtype}")
        h, w, c = t.shape
        if t.stride(2) != 1 or t.stride(1) != c or t.stride(0) < w * c:
            raise ValueError(f"image {i} must have contiguous channels and pixels (strides (>= {w * c}, {c}, 1)), got "
                             f"{t.stride()}")
        shape.append((h, w, c, t.stride(0)))
    n = len(images)
    if out is None:
        out = torch.empty((n, 3, S, S), device=images[0].device, dtype=f32)
    if (out.dtype != f32 or out.dim() != 4 or tuple(out.shape) != (n, 3, S, S) or out.stride(3) != 1
            or out.stride(2) != S or out.stride(1) != S * S or (n > 1 and out.stride(0) < 3 * S * S)):
        raise ValueError(f"out must be f32 [{n}, 3, {S}, {S}] with each image contiguous, got {tuple(out.shape)} "
                         f"{out.dtype} stride {out.stride()}")
    shape_t = torch.tensor(shape, dtype=torch.int64)
    src_t = torch.tensor([t.data_ptr() for t in images], dtype=torch.int64)
    plan_bytes, ws_bytes = ctypes.c_longlong(), ctypes.c_longlong()
    lib = L.lib()
    L.check(lib.ofk_image_plan_size(n, shape_t.data_ptr(), S, ctypes.byref(plan_bytes), ctypes.byref(ws_bytes)))
    plan = torch.empty(plan_bytes.value, dtype=torch.uint8)
    floats3 = ctypes.c_float * 3
    L.check(lib.ofk_image_plan(n, src_t.data_ptr(), shape_t.data_ptr(), S, floats3(*mean), floats3(*std),
                               plan.data_ptr(), plan_bytes.value))
    ws = torch.empty(ws_bytes.value, device=out.device, dtype=torch.uint8)
    L.check(lib.ofk_clip_preprocess(plan.data_ptr(), plan_bytes.value, ws.data_ptr(), ws_bytes.value, out.data_ptr(),
                                    out.stride(0) if n > 1 else 3 * S * S, L.stream_ptr()))
    return out


def relu_bf16(z, out=None):
    """h = relu(z) for a contiguous bf16 z (ofk_relu_bf16), exact; `out` may be z itself."""
    L.require_cuda(z, out)
    _vector(z, "z", bf16, z.numel())
    if out is None:
        out = torch.empty(z.shape, device=z.device, dtype=bf16)
    _vector(out, "out", bf16, z.numel())
    L.check(L.lib().ofk_relu_bf16(z.data_ptr(), out.data_ptr(), z.numel(), L.stream_ptr()))
    return out


def relu_bwd_bf16(dh, h, out=None):
    """dz = dh where the relu output h > 0, else 0 (ofk_relu_bwd_bf16); contiguous bf16 of one size, `out` may be dh."""
    L.require_cuda(dh, h, out)
    _vector(dh, "dh", bf16, dh.numel())
    _vector(h, "h", bf16, dh.numel())
    if out is None:
        out = torch.empty(dh.shape, device=dh.device, dtype=bf16)
    _vector(out, "out", bf16, dh.numel())
    L.check(L.lib().ofk_relu_bwd_bf16(dh.data_ptr(), h.data_ptr(), out.data_ptr(), dh.numel(), L.stream_ptr()))
    return out


def scale_bf16(x, s, out=None):
    """y = bf16(x * s) (ofk_scale_bf16) over the rows of x: bf16, 2-D or 3-D with unit inner stride and rows at one
    stride (e.g. [B, T, C] contiguous, or a column slice).  `out` (same shape, allocated when None) may be x."""
    L.require_cuda(x, out)
    if x.dtype != bf16 or x.dim() not in (2, 3) or x.stride(-1) != 1 or \
            (x.dim() == 3 and x.shape[0] > 1 and x.stride(0) != x.shape[1] * x.stride(1)):
        raise ValueError(f"x must be a bf16 [rows, C] or [B, T, C] view with unit inner stride and evenly spaced rows, "
                         f"got {tuple(x.shape)} {x.dtype} stride {x.stride()}")
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=bf16)
    if out.dtype != bf16 or out.shape != x.shape or out.stride(-1) != 1 or \
            (out.dim() == 3 and out.shape[0] > 1 and out.stride(0) != out.shape[1] * out.stride(1)):
        raise ValueError(f"out must be a bf16 view of shape {tuple(x.shape)} with unit inner stride and evenly spaced "
                         f"rows, got {tuple(out.shape)} {out.dtype} stride {out.stride()}")
    cols = x.shape[-1]
    rows = x.numel() // cols if cols else 0
    if rows:
        L.check(L.lib().ofk_scale_bf16(x.data_ptr(), x.stride(-2), rows, cols, float(s), out.data_ptr(), out.stride(-2),
                                       L.stream_ptr()))
    return out


def _seed_offset(seed_offset, p):
    if p > 0 and (seed_offset is None or seed_offset.dtype != torch.int64 or seed_offset.numel() != 2 or
                  not seed_offset.is_contiguous()):
        raise ValueError("dropout with p > 0 needs seed_offset, a contiguous int64 device tensor (seed, offset)")


def dropout_resid_fwd(x, branch, p, seed_offset, out=None):
    """out = x + dropout_p(branch) (ofk_dropout_resid_fwd): x [rows, C] f32, branch [rows, C] bf16, both with unit inner
    stride; p in [0, 1); seed_offset: int64 device (seed, offset) (unused, may be None, at p = 0).  Returns out [rows, C]
    f32 (`out`, allocated when None; may be x)."""
    L.require_cuda(x, branch, seed_offset, out)
    _rowmajor_2d(x, "x")
    _rowmajor_2d(branch, "branch")
    if x.dtype != f32 or branch.dtype != bf16 or branch.shape != x.shape:
        raise ValueError(f"x must be float32 and branch bfloat16 of one shape, got {tuple(x.shape)} {x.dtype} and "
                         f"{tuple(branch.shape)} {branch.dtype}")
    _seed_offset(seed_offset, p)
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=f32)
    _rowmajor_2d(out, "out")
    if out.dtype != f32 or out.shape != x.shape:
        raise ValueError(f"out must be float32 of shape {tuple(x.shape)}")
    rows, cols = x.shape
    if rows:
        L.check(L.lib().ofk_dropout_resid_fwd(x.data_ptr(), x.stride(0), branch.data_ptr(), branch.stride(0), rows, cols,
                                              float(p), L.ptr(seed_offset), out.data_ptr(), out.stride(0),
                                              L.stream_ptr()))
    return out


def dropout_resid_bwd(dout, p, seed_offset, out=None):
    """Gradient of dropout_resid_fwd's branch (ofk_dropout_resid_bwd): dout [rows, C] f32 with unit inner stride ->
    dbranch [rows, C] bf16 (`out`, allocated when None), from the forward's p and seed_offset."""
    L.require_cuda(dout, seed_offset, out)
    _rowmajor_2d(dout, "dout")
    if dout.dtype != f32:
        raise ValueError("dout must be float32")
    _seed_offset(seed_offset, p)
    if out is None:
        out = torch.empty(dout.shape, device=dout.device, dtype=bf16)
    _rowmajor_2d(out, "out")
    if out.dtype != bf16 or out.shape != dout.shape:
        raise ValueError(f"out must be bfloat16 of shape {tuple(dout.shape)}")
    rows, cols = dout.shape
    if rows:
        L.check(L.lib().ofk_dropout_resid_bwd(dout.data_ptr(), dout.stride(0), rows, cols, float(p),
                                              L.ptr(seed_offset), out.data_ptr(), out.stride(0), L.stream_ptr()))
    return out
