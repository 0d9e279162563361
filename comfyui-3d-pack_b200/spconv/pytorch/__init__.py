"""spconv.pytorch: SparseConvTensor, SubMConv3d and ConvAlgo on gs_b200.spconv (see the package docstring)."""
import enum

import torch
import torch.nn as nn

from gs_b200 import spconv as _sp

__all__ = ["ConvAlgo", "SparseConvTensor", "SubMConv3d", "SparseConv3d", "SparseInverseConv3d"]


class ConvAlgo(enum.Enum):
    Native = 0
    MaskImplicitGemm = 1
    MaskSplitImplicitGemm = 2


class SparseConvTensor:
    """features [N, C] over int32 indices [N, 4] = (b, x, y, z); spatial_shape [X, Y, Z] (ints or 0-d tensors).
    `features` is a property over `_features`, which TRELLIS assigns directly.  indice_dict maps an indice_key to the
    neighbour map SubMConv3d cached for these indices; replace_feature() shares it."""

    def __init__(self, features, indices, spatial_shape, batch_size, grid=None, voxel_num=None, indice_dict=None,
                 benchmark=False, permanent_thrust_allocator=False, enable_timer=False, force_algo=None):
        self._features = features
        self.indices = indices
        self.spatial_shape = [int(v) for v in spatial_shape]
        self.batch_size = int(batch_size)
        self.grid = grid
        self.voxel_num = voxel_num
        self.indice_dict = {} if indice_dict is None else indice_dict
        self.benchmark = benchmark
        self.benchmark_record = {}
        self.thrust_allocator = None
        self._timer = None
        self.force_algo = force_algo
        self.int8_scale = None

    @property
    def features(self):
        return self._features

    @features.setter
    def features(self, value):
        self._features = value

    @property
    def spatial_size(self):
        X, Y, Z = self.spatial_shape
        return X * Y * Z

    def replace_feature(self, feature):
        new = SparseConvTensor(feature, self.indices, self.spatial_shape, self.batch_size, self.grid, self.voxel_num,
                               self.indice_dict)
        new.benchmark = self.benchmark
        new.benchmark_record = self.benchmark_record
        new.thrust_allocator = self.thrust_allocator
        new._timer = self._timer
        new.force_algo = self.force_algo
        new.int8_scale = self.int8_scale
        return new

    def find_indice_pair(self, key):
        return self.indice_dict.get(key) if key is not None else None

    def dense(self, channels_first=True):
        """[B, C, X, Y, Z] (channels_first) or [B, X, Y, Z, C]; duplicate coordinates keep one row's features."""
        f = self._features.reshape(self._features.shape[0], -1)
        X, Y, Z = self.spatial_shape
        out = torch.zeros(self.batch_size, X, Y, Z, f.shape[1], dtype=f.dtype, device=f.device)
        idx = self.indices.long()
        out[idx[:, 0], idx[:, 1], idx[:, 2], idx[:, 3]] = f
        return out.permute(0, 4, 1, 2, 3).contiguous() if channels_first else out


def _triple(v, name):
    t = tuple(v) if isinstance(v, (list, tuple)) else (v, v, v)
    if len(t) != 3:
        raise ValueError(f"SubMConv3d: {name} must be an int or three ints, got {v!r}")
    return tuple(int(x) for x in t)


class SubMConv3d(nn.Module):
    """Submanifold 3D convolution: the output keeps the input's indices and row order.  weight [Cout, k, k, k, Cin]
    (spconv 2.x's layout), bias [Cout].  The neighbour map is cached in x.indice_dict[indice_key] and reused by later
    calls with the same key on the same indices tensor; without a key it is built on every call."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 indice_key=None, algo=None, fp32_accum=None, name=None):
        super().__init__()
        k = _triple(kernel_size, "kernel_size")
        if len(set(k)) != 1 or k[0] not in (1, 3):
            raise NotImplementedError(f"SubMConv3d: kernel size {kernel_size} (only 1 and 3 are implemented)")
        if _triple(stride, "stride") != (1, 1, 1):
            raise NotImplementedError("SubMConv3d: stride other than 1 is not implemented")
        if _triple(dilation, "dilation") != (1, 1, 1):
            raise NotImplementedError("SubMConv3d: dilation other than 1 is not implemented")
        if groups != 1:
            raise NotImplementedError("SubMConv3d: groups other than 1 are not implemented")
        if in_channels < 1 or out_channels < 1:
            raise ValueError(f"SubMConv3d: channel counts must be >= 1, got {in_channels}, {out_channels}")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding, self.dilation = k, (1, 1, 1), padding, (1, 1, 1)
        self.indice_key, self.algo, self.subm = indice_key, algo, True
        self.weight = nn.Parameter(torch.empty(out_channels, *k, in_channels))
        self.bias = nn.Parameter(torch.empty(out_channels)) if bias else None
        self.reset_parameters()

    def reset_parameters(self):
        fan_in = self.in_channels * self.kernel_size[0] ** 3
        bound = 1.0 / fan_in ** 0.5
        nn.init.uniform_(self.weight, -bound, bound)
        if self.bias is not None:
            nn.init.uniform_(self.bias, -bound, bound)

    def _map(self, x):
        k = self.kernel_size[0]
        key = self.indice_key
        if k == 1:                                   # a per-row GEMM: no map to build or cache
            return _sp.build_map(x.indices, x.spatial_shape, x.batch_size, 1)
        if key is not None:
            m = x.indice_dict.get(key)
            if (isinstance(m, _sp.NeighbourMap) and m.indices is x.indices and m.kernel_size == k
                    and m.spatial_shape == list(x.spatial_shape) and m.batch_size == x.batch_size):
                return m
        m = _sp.build_map(x.indices, x.spatial_shape, x.batch_size, k)
        if key is not None:
            x.indice_dict[key] = m
        return m

    def forward(self, x):
        if not isinstance(x, SparseConvTensor):
            raise TypeError(f"SubMConv3d: input must be a SparseConvTensor, got {type(x).__name__}")
        f = x.features
        if f.dim() != 2 or f.shape[1] != self.in_channels:
            raise ValueError(f"SubMConv3d: features must be [N, {self.in_channels}], got shape {tuple(f.shape)}")
        _sp.check_dtype("SubMConv3d", f)
        out = _sp.submconv3d(f, self.weight, self.bias, self._map(x))
        return x.replace_feature(out)

    def extra_repr(self):
        return f"{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}, indice_key={self.indice_key}"


class SparseConv3d(nn.Module):
    """Strided / padded sparse convolution: not implemented (no caller in the pack constructs one)."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("spconv.pytorch.SparseConv3d is not implemented: only SubMConv3d runs on the GPU "
                                  "here, and no caller in the pack builds a strided or padded sparse conv")


class SparseInverseConv3d(nn.Module):
    """Inverse sparse convolution: not implemented (no caller in the pack constructs one)."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("spconv.pytorch.SparseInverseConv3d is not implemented: only SubMConv3d runs on the "
                                  "GPU here, and no caller in the pack builds an inverse sparse conv")
