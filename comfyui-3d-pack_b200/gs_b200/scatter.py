"""Scatter reductions on the GPU: the sm_90a kernels behind gs_b200_scatter_* (include/gs_b200.h), with the argument
rules of torch_scatter 2.1's scatter_sum / scatter_add, scatter_mean and scatter_max.  The `torch_scatter` import
name (comfyui-3d-pack_b200/torch_scatter) re-exports these four.

- The index is broadcast as torch_scatter does: a negative `dim` counts from src's end, a 1-D index is unsqueezed at
  the front `dim` times, then at the end to src's rank, then expanded to src's shape (RuntimeError if it cannot be).
- With `out`, results go into its storage and the same tensor object is returned; otherwise out has src's shape with
  `dim_size` (or index.max() + 1, or 0 for an empty index) at `dim`.
- fp32 sums add src in ascending position along `dim`, one fp32 add each, starting from out's value (or +0): the
  order of torch's CPU scatter_add_, and the same bits on every run.  Mean divides that sum once by the number of
  index entries that hit the slot (at least 1).  Max replaces the running value only with a strictly greater one,
  so NaN never wins and the smallest position wins a tie; argmax is src.size(dim) where nothing won, and without
  `out` slots nothing won are 0.
- Each forward call makes one blocking device-to-host read (the index's min and max, which validate it and give
  dim_size); the backward makes none.  Work goes on the current stream.  No CPU path.
"""
import ctypes as C

import torch

from . import _lib

_CODE = {torch.float32: _lib.SCATTER_F32, torch.int32: _lib.SCATTER_I32, torch.int64: _lib.SCATTER_I64}
_SUM_DTYPES = (torch.float32, torch.int32, torch.int64)
_MEAN_DTYPES = (torch.float32,)


def _ptr(t):
    return C.c_void_p(t.data_ptr() if t is not None and t.numel() else None)


def _i64(vals):
    return (C.c_int64 * len(vals))(*vals)


def _broadcast(index, src, dim):
    if index.dim() == 1:
        for _ in range(dim):
            index = index.unsqueeze(0)
    for _ in range(index.dim(), src.dim()):
        index = index.unsqueeze(-1)
    return index.expand(src.size())


class _Call:
    """Validated arguments of one call: src, the broadcast index, out (or None), dim and dim_size."""

    def __init__(self, name, src, index, dim, out, dim_size, dtypes):
        tensors = [t for t in (src, index, out) if t is not None]
        if not all(isinstance(t, torch.Tensor) for t in tensors):
            raise TypeError(f"{name}: src, index and out must be tensors")
        if any(not t.is_cuda for t in tensors):
            raise RuntimeError(f"{name}: got a CPU tensor; gs_b200 has no CPU path (src, index and out must be CUDA tensors)")
        if any(t.device != src.device for t in tensors):
            raise RuntimeError(f"{name}: src, index and out must be on one device, got "
                               f"{', '.join(str(t.device) for t in tensors)}")
        if src.dtype not in dtypes:
            raise NotImplementedError(f"{name}: src dtype {src.dtype} is not supported; supported: "
                                      f"{', '.join(str(d) for d in dtypes)}")
        if index.dtype != torch.int64:
            raise NotImplementedError(f"{name}: index dtype {index.dtype} is not supported; supported: torch.int64")
        nd = src.dim()
        if nd < 1 or nd > _lib.SCATTER_MAX_DIMS:
            raise RuntimeError(f"{name}: src must have 1..{_lib.SCATTER_MAX_DIMS} dimensions, got {nd}")
        if not -nd <= dim < nd:
            raise IndexError(f"{name}: dim {dim} is out of range for a {nd}-D src")
        dim = dim % nd
        if dtypes is _MEAN_DTYPES and 1 < index.dim() <= dim:
            raise NotImplementedError(f"{name}: an index of 2 or more dimensions that does not reach dim {dim} is not "
                                      "supported (torch_scatter would count it along its own last dimension)")
        self.index = _broadcast(index, src, dim)
        if out is not None:
            if out.dtype != src.dtype:
                raise RuntimeError(f"{name}: out has dtype {out.dtype}, src has {src.dtype}")
            if out.dim() != nd or any(out.size(d) != src.size(d) for d in range(nd) if d != dim):
                raise RuntimeError(f"{name}: out of shape {tuple(out.shape)} does not match src {tuple(src.shape)} "
                                   f"outside dim {dim}")
            if torch._debug_has_internal_overlap(out) == 1:
                raise RuntimeError(f"{name}: out has overlapping elements (an expanded view) and cannot be written")
            dim_size = out.size(dim)
        self.name, self.src, self.out, self.dim = name, src, out, dim
        self.device, self.src_shape = src.device, tuple(src.shape)
        self.shape = _i64(list(src.shape))
        self.istr = _i64(list(self.index.stride()))
        with torch.cuda.device(src.device):
            self.dim_size = self._checked_dim_size(dim_size)

    def _checked_dim_size(self, dim_size):
        """The one host read: min and max of the index, before anything is written."""
        if dim_size is not None and int(dim_size) < 0:
            raise RuntimeError(f"{self.name}: dim_size must be >= 0, got {dim_size}")
        if self.src.numel() == 0:
            return 0 if dim_size is None else int(dim_size)
        rng = torch.empty(2, dtype=torch.int64, device=self.src.device)
        _lib.check(_lib.lib.gs_b200_scatter_index_range(self.src.dim(), self.shape, self.dim, _ptr(self.index), self.istr,
                                                        _ptr(rng), _stream()))
        lo, hi = rng.tolist()
        size = hi + 1 if dim_size is None else int(dim_size)
        bad = lo if lo < 0 else (hi if hi >= size else None)
        if bad is not None:
            raise RuntimeError(f"{self.name}: index value {bad} is out of bounds for dim_size {size}")
        return size

    def forward(self, op):
        """Runs the reduction into self.out (allocated when None); returns (out, argmax or None, scratch)."""
        src, dev = self.src, self.src.device
        has_out = self.out is not None
        out = self.out
        if out is None:
            size = list(src.shape)
            size[self.dim] = self.dim_size
            out = torch.empty(size, dtype=src.dtype, device=dev)
        nd, code = src.dim(), _CODE[src.dtype]
        nbytes = int(_lib.lib.gs_b200_scatter_scratch_bytes(op, code, nd, self.shape, self.dim, self.istr, self.dim_size))
        if nbytes == 0:
            raise RuntimeError(f"{self.name}: {_lib.last_error()}")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        argmax = torch.empty(out.shape, dtype=torch.int64, device=dev) if op == _lib.SCATTER_MAX else None
        _lib.check(_lib.lib.gs_b200_scatter_forward(op, code, nd, self.shape, self.dim, self.dim_size, _ptr(src),
                                                    _i64(list(src.stride())), _ptr(self.index), self.istr, _ptr(out),
                                                    _i64(list(out.stride())), int(has_out), _ptr(argmax), _ptr(scratch),
                                                    _stream()))
        return out, argmax, scratch


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _backward(op, call, grad, argmax, scratch, want_out):
    """(grad_src, grad_out) for the fp32 src of `call`; grad_out only for sum and mean with want_out."""
    gsrc = torch.empty(call.src_shape, dtype=torch.float32, device=call.device)
    gout = None
    if want_out and op == _lib.SCATTER_MEAN:
        gout = torch.empty(grad.shape, dtype=torch.float32, device=call.device)
    _lib.check(_lib.lib.gs_b200_scatter_backward(op, len(call.src_shape), call.shape, call.dim, call.dim_size, _ptr(call.index),
                                                 call.istr, _ptr(grad), _i64(list(grad.stride())), _ptr(argmax),
                                                 _ptr(scratch), _ptr(gsrc), _ptr(gout), _stream()))
    if want_out and op == _lib.SCATTER_SUM:
        gout = grad
    return gsrc, gout


class _ScatterFn(torch.autograd.Function):
    """One reduction (sum / mean / max) of a validated call; `out`, when given, is changed in place."""

    @staticmethod
    def forward(ctx, src, out, call, op):
        with torch.cuda.device(src.device):
            res, argmax, scratch = call.forward(op)
        call.src = call.out = None                      # the backward needs only shapes, the index and the scratch
        ctx.call, ctx.op = call, op
        ctx.has_out = out is not None
        if out is not None:
            ctx.mark_dirty(out)
        if op == _lib.SCATTER_MAX:
            ctx.mark_non_differentiable(argmax)
            ctx.save_for_backward(argmax)
            return res, argmax
        ctx.scratch = scratch if op == _lib.SCATTER_MEAN else None
        return res

    @staticmethod
    def backward(ctx, grad, *unused):
        call, op = ctx.call, ctx.op
        argmax = ctx.saved_tensors[0] if op == _lib.SCATTER_MAX else None
        want_out = ctx.has_out and ctx.needs_input_grad[1] and op != _lib.SCATTER_MAX
        with torch.cuda.device(call.device):
            gsrc, gout = _backward(op, call, grad, argmax, ctx.scratch if op == _lib.SCATTER_MEAN else None, want_out)
        return (gsrc if ctx.needs_input_grad[0] else None), gout, None, None


def _run(name, op, dtypes, src, index, dim, out, dim_size):
    call = _Call(name, src, index, dim, out, dim_size, dtypes)
    grad = torch.is_grad_enabled() and src.dtype == torch.float32 and (
        src.requires_grad or (out is not None and out.requires_grad))
    if grad:
        return _ScatterFn.apply(src, out, call, op)
    with torch.cuda.device(src.device):
        res, argmax, _ = call.forward(op)
    return (res, argmax) if op == _lib.SCATTER_MAX else res


def scatter_sum(src, index, dim=-1, out=None, dim_size=None):
    """out[..., index[i], ...] += src[..., i, ...] along `dim` (fp32, int32, int64)."""
    return _run("scatter_sum", _lib.SCATTER_SUM, _SUM_DTYPES, src, index, dim, out, dim_size)


scatter_add = scatter_sum


def scatter_mean(src, index, dim=-1, out=None, dim_size=None):
    """scatter_sum (including out's prior content), divided by the number of index entries per slot (fp32)."""
    return _run("scatter_mean", _lib.SCATTER_MEAN, _MEAN_DTYPES, src, index, dim, out, dim_size)


def scatter_max(src, index, dim=-1, out=None, dim_size=None):
    """(out, argmax int64) of the strict-greater running maximum along `dim` (fp32, int32, int64)."""
    return _run("scatter_max", _lib.SCATTER_MAX, _SUM_DTYPES, src, index, dim, out, dim_size)
