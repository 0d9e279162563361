"""Multi-head attention forward on the GPU: the sm_90a kernel behind gs_b200_attn_forward (declared in
include/gs_b200_attn.h, which states every rule), as the two calls the `flash_attn` import name
(comfyui-3d-pack_b200/flash_attn) builds on.

- varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k): q [total_q, H, 64], k / v [total_k, H, 64];
  sequence b is rows cu_seqlens[b]..cu_seqlens[b+1] (int32, B + 1 entries).  Returns [total_q, H, 64].
- dense(q, k, v): q [N, Lq, H, 64], k / v [N, Lk, H, 64].  Returns [N, Lq, H, 64].
- fp16 and bf16 (q, k, v alike); out[i] = softmax(softmax_scale * q_i . K^T) V over the row's own sequence, no mask;
  softmax_scale None means 64 ** -0.5.  A sequence without keys gives 0.  max_seqlen_q only sizes the grid.
- Inputs are read in place (packed qkv / kv slices included) when their last dim is contiguous and their strides and
  base are 16-byte aligned; others are made contiguous first.
- Argument errors are raised before any GPU work: unsupported features NotImplementedError, a dtype other than fp16 /
  bf16 or mixed dtypes TypeError, bad shapes or non-int32 cu_seqlens ValueError, CPU tensors RuntimeError.
- Every output has the same bits on every run, alone or in any batch.  Forward only: the autograd Function's backward
  raises NotImplementedError, so the forward runs in grad mode and only an actual .backward() raises.
- Work goes on the current stream; cu_seqlens is never read back to the host.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import lib, ptr, stream

HEAD_DIM = _lib.ATTN_HEAD_DIM
_DTYPES = {torch.float16: _lib.ATTN_F16, torch.bfloat16: _lib.ATTN_BF16}


def _tensor(name, arg, t):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: {arg} must be a torch.Tensor, got {type(t).__name__}")


def _dtype(name, ts):
    dt = ts[0][1].dtype
    for arg, t in ts:
        if t.dtype not in _DTYPES:
            raise TypeError(f"{name}: {arg} is {t.dtype}; only float16 and bfloat16 are implemented")
        if t.dtype != dt:
            raise TypeError(f"{name}: mixed dtypes ({ts[0][0]} {dt}, {arg} {t.dtype})")


def _heads(name, q, k, v):
    if q.size(-1) != HEAD_DIM or k.size(-1) != HEAD_DIM or v.size(-1) != HEAD_DIM:
        raise NotImplementedError(f"{name}: head dim {q.size(-1)} / {k.size(-1)} / {v.size(-1)} "
                                  f"(only {HEAD_DIM} is implemented)")
    if k.size(-2) != v.size(-2) or k.shape[:-1] != v.shape[:-1]:
        raise ValueError(f"{name}: k {tuple(k.shape)} and v {tuple(v.shape)} differ")
    if k.size(-2) != q.size(-2):
        raise NotImplementedError(f"{name}: {k.size(-2)} kv heads for {q.size(-2)} query heads "
                                  "(grouped / multi-query attention is not implemented)")


def _cu(name, arg, cu):
    _tensor(name, arg, cu)
    if cu.dtype != torch.int32:
        raise ValueError(f"{name}: {arg} must be int32, got {cu.dtype}")
    if cu.dim() != 1 or cu.numel() < 1:
        raise ValueError(f"{name}: {arg} must be 1-D with B + 1 entries, got shape {tuple(cu.shape)}")


def _cuda(name, ts, dev=None):
    for arg, t in ts:
        if not t.is_cuda:
            raise RuntimeError(f"{name}: {arg} is a CPU tensor; attention runs on CUDA tensors only")
        dev = dev or t.device
        if t.device != dev:
            raise RuntimeError(f"{name}: {arg} is on {t.device}, expected {dev}")


def _rows(t):
    """[rows, H, d] view of t with a contiguous last dim and 16-byte aligned strides and base; a copy otherwise."""
    t = t.reshape(-1, t.size(-2), t.size(-1))
    esz = t.element_size()
    if (t.stride(2) != 1 or (t.stride(0) * esz) % 16 or (t.stride(1) * esz) % 16 or t.data_ptr() % 16
            or t.stride(0) < 0 or t.stride(1) < 0):
        t = t.contiguous()
    return t


def _scale(softmax_scale):
    return HEAD_DIM ** -0.5 if softmax_scale is None else float(softmax_scale)


def _launch(q, k, v, cu_q, cu_k, max_q, max_k, B, scale):
    q3, k3, v3 = _rows(q), _rows(k), _rows(v)
    out = torch.empty(q3.shape, dtype=q.dtype, device=q.device)
    if out.numel() == 0:
        return out
    if cu_q is not None:
        cu_q, cu_k = cu_q.contiguous(), cu_k.contiguous()
    _lib.check(lib.gs_b200_attn_forward(
        _DTYPES[q.dtype], B, q3.size(1), HEAD_DIM,
        ptr(q3), q3.stride(0), q3.stride(1), ptr(k3), k3.stride(0), k3.stride(1), ptr(v3), v3.stride(0), v3.stride(1),
        ptr(cu_q), ptr(cu_k), max_q, max_k, q3.size(0), k3.size(0), C.c_float(scale), ptr(out), stream()))
    return out


class _AttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, cu_q, cu_k, max_q, max_k, B, scale):
        return _launch(q, k, v, cu_q, cu_k, max_q, max_k, B, scale)

    @staticmethod
    def backward(ctx, grad_out):
        raise NotImplementedError("gs_b200.attention: backward is not implemented (the attention kernel is "
                                  "forward only)")


def varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, softmax_scale=None,
           name="gs_b200.attention.varlen"):
    for arg, t in (("q", q), ("k", k), ("v", v)):
        _tensor(name, arg, t)
    _dtype(name, (("q", q), ("k", k), ("v", v)))
    for arg, t in (("q", q), ("k", k), ("v", v)):
        if t.dim() != 3:
            raise ValueError(f"{name}: {arg} must be [total, heads, {HEAD_DIM}], got shape {tuple(t.shape)}")
    _heads(name, q, k, v)
    _cu(name, "cu_seqlens_q", cu_seqlens_q)
    _cu(name, "cu_seqlens_k", cu_seqlens_k)
    if cu_seqlens_q.numel() != cu_seqlens_k.numel():
        raise ValueError(f"{name}: cu_seqlens_q has {cu_seqlens_q.numel()} entries, cu_seqlens_k "
                         f"{cu_seqlens_k.numel()}")
    max_q, max_k = int(max_seqlen_q), int(max_seqlen_k)
    if max_q < 0 or max_k < 0:
        raise ValueError(f"{name}: max_seqlen must be >= 0, got {max_q} / {max_k}")
    _cuda(name, (("q", q), ("k", k), ("v", v), ("cu_seqlens_q", cu_seqlens_q), ("cu_seqlens_k", cu_seqlens_k)))
    return _AttnFn.apply(q, k, v, cu_seqlens_q, cu_seqlens_k, max_q, max_k, cu_seqlens_q.numel() - 1,
                         _scale(softmax_scale))


def dense(q, k, v, softmax_scale=None, name="gs_b200.attention.dense"):
    for arg, t in (("q", q), ("k", k), ("v", v)):
        _tensor(name, arg, t)
    _dtype(name, (("q", q), ("k", k), ("v", v)))
    for arg, t in (("q", q), ("k", k), ("v", v)):
        if t.dim() != 4:
            raise ValueError(f"{name}: {arg} must be [batch, seqlen, heads, {HEAD_DIM}], got shape {tuple(t.shape)}")
    _heads(name, q, k, v)
    if k.size(0) != q.size(0):
        raise ValueError(f"{name}: batch {q.size(0)} for q, {k.size(0)} for k / v")
    _cuda(name, (("q", q), ("k", k), ("v", v)))
    N, Lq = q.shape[:2]
    out = _AttnFn.apply(q, k, v, None, None, Lq, k.size(1), N, _scale(softmax_scale))
    return out.view(q.shape)
