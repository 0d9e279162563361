"""pointnet2_ops' point-cloud operators on the GPU: the sm_90a kernels behind gs_b200_pn2_* (include/gs_b200.h, which
states every rule), as the autograd Functions pointnet2_ops.pointnet2_utils defines.  The `pointnet2_ops` import name
(comfyui-3d-pack_b200/pointnet2_ops) re-exports them.

- Float inputs are fp32 and index inputs int32 CUDA tensors, as in pointnet2_ops; read-only inputs are made
  contiguous.  A CPU tensor raises RuntimeError, another dtype TypeError, a shape mismatch or an empty point set
  (N = 0, m = 0) ValueError, all before any GPU work.
- Squared distances are ((dx*dx + dy*dy) + dz*dz) in fp32 without FMA contraction, and every tie goes to the
  smallest index, so results do not depend on the launch shape.
- furthest_point_sample, ball_query and three_nn are not differentiable.  gather_operation, grouping_operation and
  three_interpolate give grad_features only: a fold of the contributions in ascending output position with no fp32
  atomics and no host read, so the gradient has the same bits on every run.  An index outside the feature range reads
  0 in the forward and is skipped in the backward.
- Work goes on the current stream of the inputs' device.  No CPU path.
"""

import torch

from . import _lib
from ._lib import ptr, stream


def _inputs(name, **named):
    """Checks every dtype, then every device, of the (tensor, dtype) pair; returns the tensors, contiguous, in the given order."""
    for arg, (t, dtype) in named.items():
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name}: {arg} must be a torch.Tensor, got {type(t).__name__}")
        if t.dtype != dtype:
            raise TypeError(f"{name}: {arg} must be {dtype}, got {t.dtype}")
    dev = next(iter(named.values()))[0].device
    for arg, (t, _) in named.items():
        if not t.is_cuda:
            raise RuntimeError(f"{name}: {arg} is a CPU tensor; pointnet2_ops runs on CUDA tensors only")
        if t.device != dev:
            raise RuntimeError(f"{name}: {arg} is on {t.device}, expected {dev}")
    return [t.contiguous() for t, _ in named.values()]


def _shape(name, arg, t, ndim, last=None):
    if t.dim() != ndim or (last is not None and t.size(-1) != last):
        want = f"{ndim}-D" + (f" with last dimension {last}" if last is not None else "")
        raise ValueError(f"{name}: {arg} must be {want}, got shape {tuple(t.shape)}")


def _same(name, what, *pairs):
    vals = {v for _, v in pairs}
    if len(vals) > 1:
        raise ValueError(f"{name}: {what} differ: " + ", ".join(f"{a} {v}" for a, v in pairs))


def _count(name, arg, v):
    if isinstance(v, bool) or not isinstance(v, int):
        raise TypeError(f"{name}: {arg} must be an int, got {type(v).__name__}")
    if v < 0:
        raise ValueError(f"{name}: {arg} must be >= 0, got {v}")
    return v


def _nonempty(name, arg, n):
    if n == 0:
        raise ValueError(f"{name}: {arg} has no points")


class FurthestPointSampling(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, npoint):
        """xyz [B,N,3] fp32 -> int32 [B,npoint]: farthest point sampling from point 0."""
        name = "furthest_point_sample"
        npoint = _count(name, "npoint", npoint)
        (xyz,) = _inputs(name, xyz=(xyz, torch.float32))
        _shape(name, "xyz", xyz, 3, 3)
        B, N, _ = xyz.shape
        _nonempty(name, "xyz", N)
        with torch.cuda.device(xyz.device):
            out = torch.empty(B, npoint, dtype=torch.int32, device=xyz.device)
            temp = torch.empty(B * N, dtype=torch.float32, device=xyz.device) if N > _lib.PN2_FPS_ONCHIP_MAX else None
            _lib.check(_lib.lib.gs_b200_pn2_furthest_point_sample(B, N, npoint, ptr(xyz), ptr(out), ptr(temp), stream()))
        ctx.mark_non_differentiable(out)
        return out

    @staticmethod
    def backward(ctx, *grad):
        return None, None


def _gather_backward(grad, idx, B, C_, N, M):
    """grad [B,C,M] (any layout) -> grad_features [B,C,N]; entries of idx outside [0,N) fold into a discarded slot."""
    grad = grad.reshape(B, C_, M).contiguous()
    dev = grad.device
    with torch.cuda.device(dev):
        nbytes = int(_lib.lib.gs_b200_pn2_backward_scratch_bytes(B, C_, N, M, 0))
        if nbytes == 0:
            raise RuntimeError(f"gs_b200: {_lib.last_error()}")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        full = torch.empty(B, C_, N + 1, dtype=torch.float32, device=dev)
        _lib.check(_lib.lib.gs_b200_pn2_gather_backward(B, C_, N, M, ptr(grad), ptr(idx), ptr(full), ptr(scratch),
                                                        stream()))
    return full[:, :, :N]


class GatherOperation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, idx):
        """features [B,C,N] fp32, idx [B,npoint] int32 -> [B,C,npoint]."""
        name = "gather_operation"
        features, idx = _inputs(name, features=(features, torch.float32), idx=(idx, torch.int32))
        _shape(name, "features", features, 3)
        _shape(name, "idx", idx, 2)
        B, C_, N = features.shape
        _same(name, "batch sizes", ("features", B), ("idx", idx.size(0)))
        _nonempty(name, "features", N)
        M = idx.size(1)
        with torch.cuda.device(features.device):
            out = torch.empty(B, C_, M, dtype=torch.float32, device=features.device)
            _lib.check(_lib.lib.gs_b200_pn2_gather(B, C_, N, M, ptr(features), ptr(idx), ptr(out), stream()))
        ctx.save_for_backward(idx)
        ctx.dims = (B, C_, N, M)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (idx,) = ctx.saved_tensors
        return _gather_backward(grad_out, idx, *ctx.dims), None


class GroupingOperation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, idx):
        """features [B,C,N] fp32, idx [B,npoint,nsample] int32 -> [B,C,npoint,nsample]."""
        name = "grouping_operation"
        features, idx = _inputs(name, features=(features, torch.float32), idx=(idx, torch.int32))
        _shape(name, "features", features, 3)
        _shape(name, "idx", idx, 3)
        B, C_, N = features.shape
        _same(name, "batch sizes", ("features", B), ("idx", idx.size(0)))
        _nonempty(name, "features", N)
        P, S = idx.shape[1:]
        with torch.cuda.device(features.device):
            out = torch.empty(B, C_, P, S, dtype=torch.float32, device=features.device)
            _lib.check(_lib.lib.gs_b200_pn2_gather(B, C_, N, P * S, ptr(features), ptr(idx), ptr(out), stream()))
        ctx.save_for_backward(idx)
        ctx.dims = (B, C_, N, P * S)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (idx,) = ctx.saved_tensors
        return _gather_backward(grad_out, idx, *ctx.dims), None


class BallQuery(torch.autograd.Function):
    @staticmethod
    def forward(ctx, radius, nsample, xyz, new_xyz):
        """xyz [B,N,3], new_xyz [B,npoint,3] fp32 -> int32 [B,npoint,nsample]."""
        name = "ball_query"
        nsample = _count(name, "nsample", nsample)
        xyz, new_xyz = _inputs(name, xyz=(xyz, torch.float32), new_xyz=(new_xyz, torch.float32))
        _shape(name, "xyz", xyz, 3, 3)
        _shape(name, "new_xyz", new_xyz, 3, 3)
        B, N, _ = xyz.shape
        _same(name, "batch sizes", ("xyz", B), ("new_xyz", new_xyz.size(0)))
        _nonempty(name, "xyz", N)
        P = new_xyz.size(1)
        with torch.cuda.device(xyz.device):
            out = torch.zeros(B, P, nsample, dtype=torch.int32, device=xyz.device)
            _lib.check(_lib.lib.gs_b200_pn2_ball_query(B, N, P, nsample, float(radius), ptr(xyz), ptr(new_xyz),
                                                       ptr(out), stream()))
        ctx.mark_non_differentiable(out)
        return out

    @staticmethod
    def backward(ctx, *grad):
        return None, None, None, None


class ThreeNN(torch.autograd.Function):
    @staticmethod
    def forward(ctx, unknown, known):
        """unknown [B,n,3], known [B,m,3] fp32 -> (dist fp32 [B,n,3], idx int32 [B,n,3])."""
        name = "three_nn"
        unknown, known = _inputs(name, unknown=(unknown, torch.float32), known=(known, torch.float32))
        _shape(name, "unknown", unknown, 3, 3)
        _shape(name, "known", known, 3, 3)
        B, n, _ = unknown.shape
        _same(name, "batch sizes", ("unknown", B), ("known", known.size(0)))
        m = known.size(1)
        _nonempty(name, "known", m)
        with torch.cuda.device(unknown.device):
            dist = torch.empty(B, n, 3, dtype=torch.float32, device=unknown.device)
            idx = torch.empty(B, n, 3, dtype=torch.int32, device=unknown.device)
            _lib.check(_lib.lib.gs_b200_pn2_three_nn(B, n, m, ptr(unknown), ptr(known), ptr(dist), ptr(idx), stream()))
        ctx.mark_non_differentiable(dist, idx)
        return dist, idx

    @staticmethod
    def backward(ctx, *grad):
        return None, None


class ThreeInterpolate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, idx, weight):
        """features [B,C,m] fp32, idx [B,n,3] int32, weight [B,n,3] fp32 -> [B,C,n]."""
        name = "three_interpolate"
        features, idx, weight = _inputs(name, features=(features, torch.float32), idx=(idx, torch.int32),
                                        weight=(weight, torch.float32))
        _shape(name, "features", features, 3)
        _shape(name, "idx", idx, 3, 3)
        _shape(name, "weight", weight, 3, 3)
        B, C_, m = features.shape
        _same(name, "batch sizes", ("features", B), ("idx", idx.size(0)), ("weight", weight.size(0)))
        _same(name, "point counts", ("idx", idx.size(1)), ("weight", weight.size(1)))
        _nonempty(name, "features", m)
        n = idx.size(1)
        with torch.cuda.device(features.device):
            out = torch.empty(B, C_, n, dtype=torch.float32, device=features.device)
            _lib.check(_lib.lib.gs_b200_pn2_three_interpolate(B, C_, m, n, ptr(features), ptr(idx), ptr(weight),
                                                              ptr(out), stream()))
        ctx.save_for_backward(idx, weight)
        ctx.dims = (B, C_, m, n)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        idx, weight = ctx.saved_tensors
        B, C_, m, n = ctx.dims
        grad_out = grad_out.contiguous()
        dev = grad_out.device
        with torch.cuda.device(dev):
            nbytes = int(_lib.lib.gs_b200_pn2_backward_scratch_bytes(B, C_, m, n, 1))
            if nbytes == 0:
                raise RuntimeError(f"gs_b200: {_lib.last_error()}")
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            full = torch.empty(B, C_, m + 1, dtype=torch.float32, device=dev)
            _lib.check(_lib.lib.gs_b200_pn2_three_interpolate_backward(B, C_, m, n, ptr(grad_out), ptr(idx),
                                                                       ptr(weight), ptr(full), ptr(scratch), stream()))
        return full[:, :, :m], None, None


furthest_point_sample = FurthestPointSampling.apply
gather_operation = GatherOperation.apply
grouping_operation = GroupingOperation.apply
ball_query = BallQuery.apply
three_nn = ThreeNN.apply
three_interpolate = ThreeInterpolate.apply
