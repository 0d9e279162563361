"""spconv's submanifold 3D convolution on the GPU: the sm_90a kernels behind gs_b200_spconv_* (include/gs_b200.h, which
states every rule), as a neighbour-map builder and an autograd Function.  The `spconv` import name
(comfyui-3d-pack_b200/spconv) builds SubMConv3d and SparseConvTensor on them.

- indices: int32 [N, 4] rows (b, x, y, z) in any order; features [N, Cin] fp16 or fp32 (non-contiguous features are made
  contiguous); weight [Cout, k, k, k, Cin] and bias [Cout] of the features' dtype; k is 1 or 3.
- out[i] = bias + sum over offsets o in {-r..r}^3 of W[:, o + r, :] . in[row at coords(i) + o]; absent neighbours,
  neighbours outside the grid and neighbours in another batch item contribute nothing.  Duplicate coordinates resolve
  to their smallest row.  k = 1 is a per-row GEMM: every row reads its own features.
- fp16 runs on tensor cores with fp32 sums and one rounding; fp32 is true fp32 FFMA.  bf16 and fp64 raise TypeError.
- A CPU tensor raises RuntimeError, a wrong dtype TypeError, a bad shape, non-int32 indices or a spatial shape out of
  range ValueError, all before any GPU work.  Every output and gradient has the same bits on every run.
- Work goes on the current stream of the inputs' device; the map build reads nothing back to the host.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import ptr, stream

_DTYPES = {torch.float32: _lib.SPCONV_F32, torch.float16: _lib.SPCONV_F16}


def _cuda(name, arg, t):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: {arg} must be a torch.Tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise RuntimeError(f"{name}: {arg} is a CPU tensor; spconv runs on CUDA tensors only")


def spatial_dims(spatial_shape):
    """[X, Y, Z] as ints; accepts ints and 0-d tensors (TRELLIS passes list(coords.max(0)[0] + 1)[1:])."""
    try:
        dims = [int(v) for v in spatial_shape]
    except (TypeError, ValueError, RuntimeError):
        raise ValueError(f"spconv: spatial_shape must be three integers, got {spatial_shape!r}") from None
    if len(dims) != 3 or any(d < 1 for d in dims):
        raise ValueError(f"spconv: spatial_shape must be three positive integers, got {dims}")
    return dims


class NeighbourMap:
    """The k = 3 neighbour map of one indices tensor (include/gs_b200.h): nbr [N, 27] int32, mask [N] (as int32),
    sorted_keys and sorted_rows [N].  For k = 1 no map is built and every tensor is None."""

    def __init__(self, indices, spatial_shape, batch_size, kernel_size):
        self.indices, self.kernel_size = indices, kernel_size
        self.spatial_shape, self.batch_size = spatial_dims(spatial_shape), int(batch_size)
        self.nbr = self.mask = self.sorted_keys = self.sorted_rows = None


def build_map(indices, spatial_shape, batch_size, kernel_size=3):
    """Neighbour map of `indices` for a k x k x k submanifold conv, built on the device with no host read."""
    name = "spconv.build_map"
    if not isinstance(indices, torch.Tensor):
        raise TypeError(f"{name}: indices must be a torch.Tensor, got {type(indices).__name__}")
    if indices.dtype != torch.int32:
        raise ValueError(f"{name}: indices must be int32, got {indices.dtype}")
    if indices.dim() != 2 or indices.size(1) != 4:
        raise ValueError(f"{name}: indices must be [N, 4] (b, x, y, z), got shape {tuple(indices.shape)}")
    if kernel_size not in (1, 3):
        raise NotImplementedError(f"{name}: kernel size {kernel_size} (only 1 and 3 are implemented)")
    _cuda(name, "indices", indices)
    X, Y, Z = spatial_dims(spatial_shape)
    B = int(batch_size)
    if B < 1:
        raise ValueError(f"{name}: batch_size must be >= 1, got {B}")
    if B * X * Y * Z > 1 << 32:
        raise ValueError(f"{name}: batch_size * X * Y * Z = {B * X * Y * Z} exceeds 2^32")
    N = indices.size(0)
    if N > _lib.SPCONV_MAX_ROWS:
        raise ValueError(f"{name}: {N} rows (at most {_lib.SPCONV_MAX_ROWS})")
    m = NeighbourMap(indices, (X, Y, Z), B, kernel_size)
    if kernel_size == 1:
        return m
    dev = indices.device
    idx = indices.contiguous()
    if idx.data_ptr() % 16:
        idx = idx.clone()
    with torch.cuda.device(dev):
        m.nbr = torch.empty(N, 27, dtype=torch.int32, device=dev)
        m.mask = torch.empty(N, dtype=torch.int32, device=dev)
        m.sorted_keys = torch.empty(N, dtype=torch.int32, device=dev)
        m.sorted_rows = torch.empty(N, dtype=torch.int32, device=dev)
        if N:
            nbytes = int(_lib.lib.gs_b200_spconv_map_scratch_bytes(N))
            if nbytes == 0:
                raise RuntimeError(f"gs_b200: {_lib.last_error()}")
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            _lib.check(_lib.lib.gs_b200_spconv_build_map(N, B, X, Y, Z, ptr(idx), ptr(m.nbr), ptr(m.mask),
                                                         ptr(m.sorted_keys), ptr(m.sorted_rows), ptr(scratch),
                                                         stream()))
    return m


def check_dtype(name, t):
    if t.dtype not in _DTYPES:
        raise TypeError(f"{name}: features must be float16 or float32, got {t.dtype}")
    return _DTYPES[t.dtype]


class SubMConvFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, weight, bias, nmap):
        """features [N, Cin], weight [Cout, k, k, k, Cin], bias [Cout] or None, nmap from build_map -> [N, Cout]."""
        name = "spconv.SubMConv3d"
        for arg, t in (("features", features), ("weight", weight)) + ((("bias", bias),) if bias is not None else ()):
            _cuda(name, arg, t)
        dt = check_dtype(name, features)
        for arg, t in (("weight", weight),) + ((("bias", bias),) if bias is not None else ()):
            if t.dtype != features.dtype:
                raise TypeError(f"{name}: {arg} must be {features.dtype} like the features, got {t.dtype}")
        k = nmap.kernel_size
        if features.dim() != 2:
            raise ValueError(f"{name}: features must be [N, Cin], got shape {tuple(features.shape)}")
        N, Cin = features.shape
        if weight.dim() != 5 or tuple(weight.shape[1:4]) != (k, k, k) or weight.size(4) != Cin:
            raise ValueError(f"{name}: weight must be [Cout, {k}, {k}, {k}, {Cin}], got shape {tuple(weight.shape)}")
        Cout = weight.size(0)
        if bias is not None and tuple(bias.shape) != (Cout,):
            raise ValueError(f"{name}: bias must be [{Cout}], got shape {tuple(bias.shape)}")
        if N != nmap.indices.size(0):
            raise ValueError(f"{name}: {N} feature rows for {nmap.indices.size(0)} indices")
        if Cin < 1 or Cout < 1:
            raise ValueError(f"{name}: channel counts must be >= 1, got Cin {Cin}, Cout {Cout}")
        if features.device != weight.device or features.device != nmap.indices.device:
            raise RuntimeError(f"{name}: features, weight and indices must be on one device")
        features, weight = features.contiguous(), weight.contiguous()
        bias = bias.contiguous() if bias is not None else None
        dev = features.device
        with torch.cuda.device(dev):
            out = torch.empty(N, Cout, dtype=features.dtype, device=dev)
            if N:
                _lib.check(_lib.lib.gs_b200_spconv_forward(dt, N, Cin, Cout, k, ptr(features), ptr(nmap.nbr),
                                                           ptr(nmap.mask), ptr(weight), ptr(bias), ptr(out),
                                                           stream()))
        ctx.save_for_backward(features, weight)
        ctx.nmap, ctx.dt, ctx.has_bias = nmap, dt, bias is not None
        return out

    @staticmethod
    def backward(ctx, grad_out):
        features, weight = ctx.saved_tensors
        nmap, dt = ctx.nmap, ctx.dt
        k = nmap.kernel_size
        N, Cin = features.shape
        Cout = weight.size(0)
        grad_out = grad_out.contiguous().to(features.dtype)
        dev = features.device
        need_x, need_w, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2] and ctx.has_bias
        gx = gw = gb = None
        with torch.cuda.device(dev):
            nbytes = int(_lib.lib.gs_b200_spconv_backward_scratch_bytes(dt, N, Cin, Cout, k))
            if nbytes == 0:
                raise RuntimeError(f"gs_b200: {_lib.last_error()}")
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            if need_x:
                gx = torch.empty(N, Cin, dtype=features.dtype, device=dev)
                _lib.check(_lib.lib.gs_b200_spconv_dgrad(dt, N, Cin, Cout, k, ptr(grad_out), ptr(nmap.nbr),
                                                         ptr(nmap.mask), ptr(nmap.sorted_keys),
                                                         ptr(nmap.sorted_rows), ptr(weight), ptr(gx),
                                                         ptr(scratch), stream()))
            if need_w or need_b:
                gw = torch.empty_like(weight) if need_w else None
                gb = torch.empty(Cout, dtype=weight.dtype, device=dev) if need_b else None
                _lib.check(_lib.lib.gs_b200_spconv_wgrad(dt, N, Cin, Cout, k, ptr(features), ptr(grad_out),
                                                         ptr(nmap.nbr), C.c_void_p(gw.data_ptr() if gw is not None else None),
                                                         C.c_void_p(gb.data_ptr() if gb is not None else None),
                                                         ptr(scratch), stream()))
        return gx, gw, gb, None


def submconv3d(features, weight, bias, nmap):
    """Submanifold conv of `features` over the rows of `nmap` (build_map); differentiable in features, weight, bias."""
    return SubMConvFunction.apply(features, weight, bias, nmap)
