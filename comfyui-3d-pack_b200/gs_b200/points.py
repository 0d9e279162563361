"""pytorch3d's point rasterizer and TriplaneGaussian's points_projection on the GPU: the sm_90a kernels behind
gs_b200_pts_* (declared in include/gs_b200_pts.h, which states every rule), under the names TriplaneGaussian
imports from pytorch3d (`utils/ops.py`, `models/snowflake/model_spdpp.py`).  This is a module, not a `pytorch3d`
package: callers take it in by changing their import lines.

- PointsRasterizationSettings, Pointclouds, cameras_from_opencv_projection and PointsRasterizer follow pytorch3d 0.7's
  signatures where TriplaneGaussian uses them; the rasterizer returns PointFragments(idx, zbuf, dists) as pytorch3d's.
  `bin_size` and `max_points_per_bin` are accepted and ignored: the kernels bin by point whatever they say.
- Conventions (pytorch3d's): NDC +X left, +Y up, the shorter image side spanning [-1, 1]; z is the view-space depth.
  A point is drawn only when z > 0.  A point covers a pixel iff its squared NDC distance to the pixel centre is
  below radius^2 (fp32, strict); each pixel keeps its points_per_pixel (1..8) covering points nearest in z, ties to
  the smaller packed index.
- points_projection lifts the feature map onto the points: a point takes the features of the largest linear pixel
  index (b, y, x, k) that selected it (what a sequential index_put leaves), 0 when no pixel did.  Its backward to
  local_features is the exact adjoint of that: each winning pixel receives its point's gradient (slots summed in
  order), with no atomics, the same bits on every run.  No gradient reaches points or cameras.
- Points are fp32 CUDA tensors.  A CPU tensor raises RuntimeError, another points dtype TypeError, points_per_pixel
  outside [1, 8] NotImplementedError and a shape mismatch ValueError, all before any GPU work.  Work goes on the
  current stream of the points' device; no output size depends on the data, so nothing is read back to the host.
- CamerasBase, AlphaCompositor, NormWeightedCompositor and PointsRenderer exist so the import lines resolve; building
  one raises NotImplementedError.
"""

import ctypes as C
import dataclasses
from typing import NamedTuple, Optional, Sequence, Union

import torch

from . import _lib
from ._lib import lib, ptr, stream

MAX_K = _lib.PTS_MAX_K


class PointFragments(NamedTuple):
    idx: torch.Tensor    # int32 [N, H, W, K]: packed point index, -1 where empty
    zbuf: torch.Tensor   # fp32 [N, H, W, K]: view-space z, -1 where empty
    dists: torch.Tensor  # fp32 [N, H, W, K]: squared NDC distance to the pixel centre, -1 where empty


@dataclasses.dataclass
class PointsRasterizationSettings:
    image_size: Union[int, Sequence[int]] = 256
    radius: float = 0.01
    points_per_pixel: int = 8
    bin_size: Optional[int] = None
    max_points_per_bin: Optional[int] = None


def _tensor(name, arg, t):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: {arg} must be a torch.Tensor, got {type(t).__name__}")
    return t


def _cuda(name, arg, t, dev=None):
    if not t.is_cuda:
        raise RuntimeError(f"{name}: {arg} is a CPU tensor; the point rasterizer runs on CUDA tensors only")
    if dev is not None and t.device != dev:
        raise RuntimeError(f"{name}: {arg} is on {t.device}, expected {dev}")


def _points(name, arg, t, ndim):
    _tensor(name, arg, t)
    if t.dtype != torch.float32:
        raise TypeError(f"{name}: {arg} must be torch.float32, got {t.dtype}")
    _cuda(name, arg, t)
    if t.dim() != ndim or t.size(-1) != 3:
        raise ValueError(f"{name}: {arg} must be {ndim}-D with last dimension 3, got shape {tuple(t.shape)}")


def _floating(name, arg, t, shape, dev):
    """A float tensor of `shape` (None = any size) on `dev`."""
    _tensor(name, arg, t)
    if not t.is_floating_point():
        raise TypeError(f"{name}: {arg} must be a floating-point tensor, got {t.dtype}")
    _cuda(name, arg, t, dev)
    if t.dim() != len(shape) or any(s is not None and t.size(i) != s for i, s in enumerate(shape)):
        want = "[" + ", ".join("*" if s is None else str(s) for s in shape) + "]"
        raise ValueError(f"{name}: {arg} must have shape {want}, got {tuple(t.shape)}")


class Pointclouds:
    """pytorch3d's Pointclouds for `points` only: a list of [P_i, 3] tensors or a padded [N, P, 3] tensor (every cloud
    then has P points).  Packed point indices run over the clouds in order."""

    def __init__(self, points, normals=None, features=None):
        name = "Pointclouds"
        if normals is not None or features is not None:
            raise NotImplementedError(f"{name}: normals and features are not supported")
        if isinstance(points, torch.Tensor):
            _points(name, "points", points, 3)
            self._padded, self._list = points, None
            self._lens = [points.size(1)] * points.size(0)
            self.device = points.device
        elif isinstance(points, (list, tuple)):
            for i, p in enumerate(points):
                _points(name, f"points[{i}]", p, 2)
                _cuda(name, f"points[{i}]", p, points[0].device)
            if not points:
                raise ValueError(f"{name}: an empty list has no device; pass a [0, P, 3] tensor instead")
            self._padded, self._list = None, list(points)
            self._lens = [p.size(0) for p in points]
            self.device = points[0].device
        else:
            raise TypeError(f"{name}: points must be a list of tensors or a tensor, got {type(points).__name__}")

    def __len__(self):
        return len(self._lens)

    def isempty(self):
        return len(self._lens) == 0 or sum(self._lens) == 0

    def points_list(self):
        return self._list if self._list is not None else list(self._padded.unbind(0))

    def points_packed(self):
        if self._list is None:
            return self._padded.reshape(-1, 3)
        return torch.cat(self._list, 0)

    def points_padded(self):
        if self._list is None:
            return self._padded
        out = torch.zeros(len(self._lens), max(self._lens), 3, dtype=torch.float32, device=self.device)
        for i, p in enumerate(self._list):
            out[i, :p.size(0)] = p
        return out

    def num_points_per_cloud(self):
        return torch.tensor(self._lens, dtype=torch.int64, device=self.device)

    def cloud_to_packed_first_idx(self):
        first = [0]
        for n in self._lens[:-1]:
            first.append(first[-1] + n)
        return torch.tensor(first, dtype=torch.int64, device=self.device)


class CamerasBase:
    """Named for model_spdpp.py's import block; only cameras_from_opencv_projection's cameras are built here."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("gs_b200.points: only cameras_from_opencv_projection's cameras are supported")


class OpenCVCameras(CamerasBase):
    """What cameras_from_opencv_projection returns: OpenCV's world-to-camera R [N,3,3] and tvec [N,3], the pixel-space
    camera matrix [N,3,3] and image_size [N,2] = (height, width), kept as given (fp32) and applied in the kernel."""

    def __init__(self, R, tvec, camera_matrix, image_size):  # noqa: super().__init__ raises by design
        self.R, self.T, self.camera_matrix, self.image_size = R, tvec, camera_matrix, image_size
        self.device = R.device

    def __len__(self):
        return self.R.size(0)


def cameras_from_opencv_projection(R, tvec, camera_matrix, image_size):
    """pytorch3d.utils.cameras_from_opencv_projection: R [N,3,3], tvec [N,3], camera_matrix [N,3,3] (float CUDA
    tensors), image_size [N,2] = (height, width) -> cameras for PointsRasterizer."""
    name = "cameras_from_opencv_projection"
    _floating(name, "R", R, (None, 3, 3), None)
    dev, N = R.device, R.size(0)
    _floating(name, "tvec", tvec, (N, 3), dev)
    _floating(name, "camera_matrix", camera_matrix, (N, 3, 3), dev)
    _tensor(name, "image_size", image_size)
    _cuda(name, "image_size", image_size, dev)
    if image_size.dim() != 2 or tuple(image_size.shape) != (N, 2):
        raise ValueError(f"{name}: image_size must have shape [{N}, 2], got {tuple(image_size.shape)}")
    f32 = lambda t: t.detach().to(torch.float32).contiguous()  # noqa: E731
    return OpenCVCameras(f32(R), f32(tvec), f32(camera_matrix), f32(image_size))


def _settings(name, s):
    if not isinstance(s, PointsRasterizationSettings):
        raise TypeError(f"{name}: raster_settings must be PointsRasterizationSettings, got {type(s).__name__}")
    size = s.image_size
    hw = (size, size) if isinstance(size, int) and not isinstance(size, bool) else tuple(size) if isinstance(size, (tuple, list)) else None
    if hw is None or len(hw) != 2 or any(isinstance(v, bool) or not isinstance(v, int) or v < 1 for v in hw):
        raise ValueError(f"{name}: image_size must be a positive int or (H, W), got {size!r}")
    K = s.points_per_pixel
    if isinstance(K, bool) or not isinstance(K, int):
        raise TypeError(f"{name}: points_per_pixel must be an int, got {type(K).__name__}")
    if not 1 <= K <= MAX_K:
        raise NotImplementedError(f"{name}: points_per_pixel {K} is outside the supported 1..{MAX_K}")
    r = s.radius
    if isinstance(r, torch.Tensor):
        raise NotImplementedError(f"{name}: a per-point radius tensor is not supported; pass a float")
    if isinstance(r, bool) or not isinstance(r, (int, float)):
        raise TypeError(f"{name}: radius must be a float, got {type(r).__name__}")
    if not r >= 0:
        raise ValueError(f"{name}: radius must be >= 0, got {r}")
    return hw[0], hw[1], K, float(r)


def _rasterize(N, packed, first, R, T, Km, hw_t, H, W, K, radius, fragments):
    """idx (and zbuf / dists when `fragments`) for N clouds; launches on the current stream of packed's device."""
    dev = packed.device
    P = packed.size(0)
    idx = torch.empty(N, H, W, K, dtype=torch.int32, device=dev)
    zbuf = torch.empty(N, H, W, K, dtype=torch.float32, device=dev) if fragments else None
    dists = torch.empty(N, H, W, K, dtype=torch.float32, device=dev) if fragments else None
    nbytes = int(lib.gs_b200_pts_scratch_bytes(N, P, H, W, K))
    if nbytes == 0:
        raise RuntimeError(f"gs_b200: {_lib.last_error()}")
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    _lib.check(lib.gs_b200_pts_rasterize(N, P, H, W, K, radius, R.size(0), ptr(packed), ptr(first), ptr(R), ptr(T),
                                         ptr(Km), ptr(hw_t), ptr(idx), ptr(zbuf), ptr(dists), ptr(scratch), stream()))
    return idx, zbuf, dists


class PointsRasterizer(torch.nn.Module):
    """pytorch3d's PointsRasterizer for cameras_from_opencv_projection's cameras: forward(point_clouds) ->
    PointFragments.  `cameras` and `raster_settings` may also be passed to the call, as in pytorch3d."""

    def __init__(self, cameras=None, raster_settings=None):
        super().__init__()
        self.cameras = cameras
        self.raster_settings = raster_settings if raster_settings is not None else PointsRasterizationSettings()

    def forward(self, point_clouds, **kwargs):
        name = "PointsRasterizer"
        cameras = kwargs.get("cameras", self.cameras)
        H, W, K, radius = _settings(name, kwargs.get("raster_settings", self.raster_settings))
        if not isinstance(point_clouds, Pointclouds):
            raise TypeError(f"{name}: expected gs_b200.points.Pointclouds, got {type(point_clouds).__name__}")
        if cameras is None:
            raise ValueError(f"{name}: cameras were not given")
        if not isinstance(cameras, OpenCVCameras):
            raise NotImplementedError(f"{name}: only cameras_from_opencv_projection's cameras are supported")
        N, dev = len(point_clouds), point_clouds.device
        if cameras.device != dev:
            raise RuntimeError(f"{name}: cameras are on {cameras.device}, point clouds on {dev}")
        if len(cameras) not in (1, N):
            raise ValueError(f"{name}: {len(cameras)} cameras for {N} point clouds (need 1 or {N})")
        with torch.cuda.device(dev):
            packed = point_clouds.points_packed().contiguous()
            first = None if point_clouds._list is None else point_clouds.cloud_to_packed_first_idx()
            if first is not None:
                first = torch.cat([first, torch.full((1,), packed.size(0), dtype=torch.int64, device=dev)])
            return PointFragments(*_rasterize(N, packed, first, cameras.R, cameras.T, cameras.camera_matrix,
                                              cameras.image_size, H, W, K, radius, True))


class _Lift(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, idx, P):
        """features [N,C,H,W] fp32 (any strides), idx int32 [N,H,W,K] -> [P, C] fp32."""
        N, C_, H, W = features.shape
        K = idx.size(3)
        dev = features.device
        winner = torch.empty(P, dtype=torch.int32, device=dev)
        out = torch.empty(P, C_, dtype=torch.float32, device=dev)
        strides = (C.c_int64 * 4)(*features.stride())
        _lib.check(lib.gs_b200_pts_lift(N, P, H, W, K, C_, ptr(idx), ptr(features), strides, ptr(winner), ptr(out),
                                        stream()))
        ctx.save_for_backward(idx, winner)
        ctx.dims = (N, P, H, W, K, C_)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        idx, winner = ctx.saved_tensors
        N, P, H, W, K, C_ = ctx.dims
        grad_out = grad_out.to(torch.float32).contiguous()
        with torch.cuda.device(grad_out.device):
            grad = torch.empty(N, C_, H, W, dtype=torch.float32, device=grad_out.device)
            _lib.check(lib.gs_b200_pts_lift_backward(N, P, H, W, K, C_, ptr(idx), ptr(winner), ptr(grad_out), ptr(grad),
                                                     stream()))
        return grad, None, None


def points_projection(points, c2ws, intrinsics, local_features, raster_point_radius: float = 0.0075,
                      raster_points_per_pixel: int = 1, bin_size: int = 0):
    """TriplaneGaussian's points_projection (utils/ops.py), fused: points [B,Np,3] fp32, c2ws [B,4,4] camera-to-world
    (OpenCV axes), intrinsics [B,3,3] in pixels, local_features [B,C,H,W] -> [B,Np,C] fp32, each point carrying the
    features of the last pixel (largest (b, y, x, k)) that selected it and 0 when none did.  One camera for every
    cloud is also accepted (c2ws [1,4,4], intrinsics [1,3,3]).  Differentiable in local_features only."""
    name = "points_projection"
    _points(name, "points", points, 3)
    dev = points.device
    B, Np, _ = points.shape
    _tensor(name, "local_features", local_features)
    if not local_features.is_floating_point():
        raise TypeError(f"{name}: local_features must be a floating-point tensor, got {local_features.dtype}")
    _cuda(name, "local_features", local_features, dev)
    if local_features.dim() != 4 or local_features.size(0) != B:
        raise ValueError(f"{name}: local_features must be [{B}, C, H, W], got {tuple(local_features.shape)}")
    _floating(name, "c2ws", c2ws, (None, 4, 4), dev)
    ncam = c2ws.size(0)
    if ncam not in (1, B):
        raise ValueError(f"{name}: {ncam} cameras for {B} point clouds (need 1 or {B})")
    _floating(name, "intrinsics", intrinsics, (ncam, 3, 3), dev)
    _, C_, H, W = local_features.shape
    settings = PointsRasterizationSettings(image_size=(H, W), radius=raster_point_radius,
                                           points_per_pixel=raster_points_per_pixel, bin_size=bin_size)
    H, W, K, radius = _settings(name, settings)
    with torch.cuda.device(dev):
        w2cs = torch.linalg.inv_ex(c2ws.detach())[0]          # torch.inverse without its host-side error check
        f32 = lambda t: t.to(torch.float32).contiguous()       # noqa: E731
        idx, _, _ = _rasterize(B, points.reshape(B * Np, 3).contiguous(), None, f32(w2cs[:, :3, :3]), f32(w2cs[:, :3, 3]),
                               f32(intrinsics.detach()), None, H, W, K, radius, False)
        out = _Lift.apply(local_features.to(torch.float32), idx, B * Np)
    return out.reshape(B, Np, C_)


class _Unsupported:
    def __init__(self, *args, **kwargs):
        raise NotImplementedError(f"gs_b200.points: {type(self).__name__} is not implemented (only the point "
                                  "rasterizer and points_projection are)")


class AlphaCompositor(_Unsupported):
    pass


class NormWeightedCompositor(_Unsupported):
    pass


class PointsRenderer(_Unsupported):
    pass
