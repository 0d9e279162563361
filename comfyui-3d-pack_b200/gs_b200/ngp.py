"""Host-side mirror of the kiui.gridencoder / kiui.nn / nerfacc surface used by the reference's Instant-NGP node
(MVs_Algorithms/NeRF/Instant_NGP.py:20-35,101-156,195; LGM/nerf_marching_cubes_converter.py:56-59,98-154).
Compute is the sm_90a library behind include/ngp_b200.h; PyTorch is memory, autograd glue, and the tiny
MLPs (plain library GEMMs).  No CPU path."""
import ctypes as C
import math

import numpy as np
import torch
import torch.nn as nn

from . import _lib

_P = lambda t: None if t is None else C.c_void_p(t.data_ptr())


_RNG = None


def set_rng(generator=None):
    """Reproducibility hook: with a CPU torch.Generator set, the three random draws of this module (occupancy-grid
    update jitter, stratified sampling offsets, TV sample points) come from it (drawn on the CPU, moved to the device)
    instead of the device RNG — this is how tests replay a CPU-generated reference run on the GPU.  None restores the default."""
    global _RNG
    _RNG = generator


def _rand(shape, device):
    if _RNG is None:
        return torch.rand(shape, device=device, dtype=torch.float32)
    return torch.rand(shape, generator=_RNG, dtype=torch.float32).to(device)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _f32c(t):
    if not t.is_cuda:
        raise RuntimeError("CUDA tensor required (gs_b200 NGP ops have no CPU path)")
    t = t.detach()
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


# ------------------------------------------------------------------------------------------------ grid encoder
class _GridEncode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, emb, enc):
        xs = _f32c(x); e = _f32c(emb)
        N = xs.shape[0]
        out = torch.empty(N, enc.num_levels * enc.level_dim, device=xs.device)
        with torch.cuda.device(xs.device):
            _lib.check(_lib.lib.ngp_b200_grid_encode_fwd(_P(xs), N, _P(e), enc._off_ptr, enc.num_levels, float(enc._bound_call),
                                                         float(enc.per_level_scale), int(enc.base_resolution), _P(out), _stream()))
        ctx.save_for_backward(xs)
        ctx.enc = enc
        ctx.bound = float(enc._bound_call)
        ctx.shape = emb.shape
        return out

    @staticmethod
    def backward(ctx, g):
        (xs,) = ctx.saved_tensors
        enc = ctx.enc
        g = _f32c(g)
        d_emb = torch.zeros(ctx.shape, device=xs.device)
        with torch.cuda.device(xs.device):
            _lib.check(_lib.lib.ngp_b200_grid_encode_bwd(_P(xs), xs.shape[0], enc._off_ptr, enc.num_levels, ctx.bound,
                                                         float(enc.per_level_scale), int(enc.base_resolution), _P(g), _P(d_emb), _stream()))
        return None, d_emb, None


class GridEncoder(nn.Module):
    """kiui.gridencoder.GridEncoder (torch-ngp): defaults as the package (SURVEY App. A.3); the reference passes
    num_levels=12 (Instant_NGP.py:32-33).  Only the configuration the reference can reach is implemented:
    input_dim=3, level_dim=2, gridtype='hash', align_corners=False, interpolation='linear'."""

    def __init__(self, input_dim=3, num_levels=16, level_dim=2, per_level_scale=2, base_resolution=16, log2_hashmap_size=19,
                 desired_resolution=None, gridtype="hash", align_corners=False, interpolation="linear"):
        super().__init__()
        if desired_resolution is not None:
            per_level_scale = np.exp2(np.log2(desired_resolution / base_resolution) / (num_levels - 1))
        if input_dim != 3 or level_dim != 2 or gridtype != "hash" or align_corners or interpolation != "linear":
            raise NotImplementedError("gs_b200 GridEncoder: input_dim=3, level_dim=2, hash, align_corners=False, linear only")
        self.input_dim, self.num_levels, self.level_dim = input_dim, num_levels, level_dim
        self.per_level_scale, self.base_resolution, self.log2_hashmap_size = per_level_scale, base_resolution, log2_hashmap_size
        self.output_dim = num_levels * level_dim
        self.max_params = 2 ** log2_hashmap_size
        offsets, offset = [], 0
        for i in range(num_levels):
            resolution = int(np.ceil(base_resolution * per_level_scale ** i))
            params_in_level = min(self.max_params, (resolution + 1) ** input_dim)
            params_in_level = int(np.ceil(params_in_level / 8) * 8)
            offsets.append(offset); offset += params_in_level
        offsets.append(offset)
        self._offsets_np = np.array(offsets, dtype=np.int32)
        self._off_ptr = C.c_void_p(self._offsets_np.ctypes.data)
        self.register_buffer("offsets", torch.from_numpy(self._offsets_np.copy()))
        self.n_params = offsets[-1] * level_dim
        self.embeddings = nn.Parameter(torch.empty(offset, level_dim))
        self._bound_call = 1.0
        self.reset_parameters()

    def reset_parameters(self):
        self.embeddings.data.uniform_(-1e-4, 1e-4)

    def forward(self, inputs, bound=1):
        prefix = list(inputs.shape[:-1])
        x = inputs.reshape(-1, self.input_dim)
        self._bound_call = float(bound)
        out = _GridEncode.apply(x, self.embeddings, self)
        return out.view(prefix + [self.output_dim])

    @torch.no_grad()
    def grad_total_variation(self, weight=1e-7, inputs=None, bound=1, B=1000000):
        if self.embeddings.grad is None:
            raise ValueError("grad is None, should be called after loss.backward() and before optimizer.step()!")
        dev = self.embeddings.device
        if inputs is None:
            inputs = _rand((B, self.input_dim), dev) * 2 * bound - bound               # uniform in [-bound, bound]
        x = _f32c(inputs.reshape(-1, self.input_dim))
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.ngp_b200_grid_tv_grad(_P(x), x.shape[0], _P(_f32c(self.embeddings)), self._off_ptr, self.num_levels,
                                                      float(bound), float(self.per_level_scale), int(self.base_resolution),
                                                      float(weight), _P(self.embeddings.grad), _stream()))


# ------------------------------------------------------------------------------------------------ kiui.nn / kiui.op / kiui.cam
class _FusedMLP2(torch.autograd.Function):
    """y = W2 relu(W1 x): one pass, hidden layer in registers (ngp_mlp.cu); backward recomputes it."""

    @staticmethod
    def forward(ctx, x, W1, W2):
        xs, w1, w2 = _f32c(x), _f32c(W1), _f32c(W2)
        N, Din = xs.shape
        H, Dout = w1.shape[0], w2.shape[0]
        y = torch.empty(N, Dout, device=xs.device)
        with torch.cuda.device(xs.device):
            _lib.check(_lib.lib.ngp_b200_mlp2_fwd(_P(xs), N, Din, H, Dout, _P(w1), _P(w2), _P(y), _stream()))
        ctx.save_for_backward(xs, w1, w2)
        ctx.need_gx = x.requires_grad
        return y

    @staticmethod
    def backward(ctx, gy):
        xs, w1, w2 = ctx.saved_tensors
        N, Din = xs.shape
        H, Dout = w1.shape[0], w2.shape[0]
        g = _f32c(gy)
        gx = torch.empty_like(xs) if ctx.need_gx else None
        gw1 = torch.zeros_like(w1); gw2 = torch.zeros_like(w2)
        with torch.cuda.device(xs.device):
            _lib.check(_lib.lib.ngp_b200_mlp2_bwd(_P(xs), N, Din, H, Dout, _P(w1), _P(w2), _P(g), _P(gx), _P(gw1), _P(gw2), _stream()))
        return gx, gw1, gw2


class MLP(nn.Module):
    """kiui.nn.MLP: Linear(+ReLU) stack.  The 2-layer, bias-free, hidden-32 shape the reference uses
    (Instant_NGP.py:34-35) runs as ONE fused kernel; any other shape uses torch Linear (library GEMM)."""

    def __init__(self, dim_in, dim_out, dim_hidden, num_layers, bias=True):
        super().__init__()
        self.dim_in, self.dim_out, self.dim_hidden, self.num_layers = dim_in, dim_out, dim_hidden, num_layers
        self.net = nn.ModuleList([nn.Linear(dim_in if l == 0 else dim_hidden, dim_out if l == num_layers - 1 else dim_hidden, bias=bias)
                                  for l in range(num_layers)])

    def _fusable(self, x):
        return (self.num_layers == 2 and self.net[0].bias is None and x.is_cuda and x.dtype == torch.float32 and x.dim() == 2
                and x.shape[0] > 0 and _lib.lib.ngp_b200_mlp2_supported(self.dim_in, self.dim_hidden, self.dim_out))

    def forward(self, x):
        if self._fusable(x):
            return _FusedMLP2.apply(x, self.net[0].weight, self.net[1].weight)
        for l in range(self.num_layers):
            x = self.net[l](x)
            if l != self.num_layers - 1:
                x = torch.nn.functional.relu(x, inplace=True)
        return x


class _TruncExp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * torch.exp(x.clamp(max=15))


trunc_exp = _TruncExp.apply


def inverse_sigmoid(x, eps=1e-6):
    x = torch.clamp(x, eps, 1 - eps) if isinstance(x, torch.Tensor) else np.clip(x, eps, 1 - eps)
    return torch.log(x / (1 - x)) if isinstance(x, torch.Tensor) else np.log(x / (1 - x))


def safe_normalize(x, eps=1e-20):
    if isinstance(x, np.ndarray):
        return x / np.sqrt(np.maximum(np.sum(x * x, axis=-1, keepdims=True), eps))
    return x / torch.sqrt(torch.clamp(torch.sum(x * x, -1, keepdim=True), min=eps))


# ------------------------------------------------------------------------------------------------ nerfacc
class OccGridEstimator(nn.Module):
    """nerfacc.OccGridEstimator for a single level (the reference passes levels=1, Instant_NGP.py:30)."""

    def __init__(self, roi_aabb, resolution=128, levels=1):
        super().__init__()
        if levels != 1:
            raise NotImplementedError("levels != 1 is not used by the reference")
        aabb = torch.as_tensor(roi_aabb, dtype=torch.float32).flatten()
        self.register_buffer("aabbs", aabb[None].clone())
        self.resolution = int(resolution)
        R = self.resolution
        self.cells_per_lvl = R ** 3
        self.register_buffer("occs", torch.zeros(R ** 3, device=aabb.device))
        self.register_buffer("binaries", torch.zeros(1, R, R, R, dtype=torch.bool, device=aabb.device))
        g = torch.arange(R)
        coords = torch.stack(torch.meshgrid(g, g, g, indexing="ij"), dim=-1).reshape(-1, 3)
        self.register_buffer("grid_coords", coords.to(aabb.device))
        self.register_buffer("grid_indices", torch.arange(R ** 3, device=aabb.device))

    @torch.no_grad()
    def update_every_n_steps(self, step, occ_eval_fn, occ_thre=1e-2, ema_decay=0.95, warmup_steps=256, n=16):
        if not self.training:
            raise RuntimeError("You should only call this function only during training.")
        if step % n == 0 and self.training:
            self._update(step, occ_eval_fn, occ_thre, ema_decay, warmup_steps)

    @torch.no_grad()
    def mark_invisible_cells(self, *a, **k):
        raise NotImplementedError

    @torch.no_grad()
    def _update(self, step, occ_eval_fn, occ_thre, ema_decay, warmup_steps):
        R = self.resolution
        dev = self.occs.device
        if step < warmup_steps:
            indices = self.grid_indices
        else:
            N = self.cells_per_lvl // 4
            uniform = torch.randint(self.cells_per_lvl, (N,), device=dev)
            occupied = torch.nonzero(self.binaries.flatten())[:, 0]
            if N < len(occupied):
                occupied = occupied[torch.randint(len(occupied), (N,), device=dev)]
            indices = torch.cat([uniform, occupied], dim=0)
        coords = self.grid_coords[indices]
        x = (coords + _rand(tuple(coords.shape), coords.device)) / R
        lo, hi = self.aabbs[0, :3], self.aabbs[0, 3:]
        x = lo + x * (hi - lo)
        occ = occ_eval_fn(x).squeeze(-1)
        self.occs[indices] = torch.maximum(self.occs[indices] * ema_decay, occ)
        thre = torch.clamp(self.occs[self.occs >= 0].mean(), max=occ_thre)
        self.binaries = (self.occs > thre).view(self.binaries.shape)

    @torch.no_grad()
    def sampling(self, rays_o, rays_d, sigma_fn=None, alpha_fn=None, near_plane=0.0, far_plane=1e10, t_min=None, t_max=None,
                 render_step_size=1e-3, early_stop_eps=1e-4, alpha_thre=0.0, stratified=False, cone_angle=0.0):
        if cone_angle != 0.0 or t_min is not None or t_max is not None or alpha_fn is not None:
            raise NotImplementedError("cone_angle / t_min / t_max / alpha_fn are not used by the reference")
        ro = _f32c(rays_o); rd = _f32c(rays_d)
        n = ro.shape[0]
        t_off = _rand((n,), ro.device) * render_step_size if stratified else None
        ray_indices, t_starts, t_ends = march_rays(ro, rd, self.binaries[0], self.aabbs[0], near_plane, far_plane,
                                                   render_step_size, t_off)
        if (alpha_thre > 0.0 or early_stop_eps > 0.0) and sigma_fn is not None and ray_indices.numel() > 0:
            alpha_thre = min(alpha_thre, float(self.occs.mean()))
            sigmas = sigma_fn(t_starts, t_ends, ray_indices)
            w, trans, alphas = render_weight_from_density(t_starts, t_ends, sigmas.detach(), ray_indices=ray_indices, n_rays=n)
            masks = (trans >= early_stop_eps) & (alphas >= alpha_thre)
            ray_indices, t_starts, t_ends = ray_indices[masks], t_starts[masks], t_ends[masks]
        return ray_indices, t_starts, t_ends


@torch.no_grad()
def march_rays(rays_o, rays_d, binary, aabb, near_plane, far_plane, dt, t_offset=None):
    """Packed samples (ray_indices int64 sorted, t_starts, t_ends) — fixed-step marching with empty-space skipping."""
    ro = _f32c(rays_o); rd = _f32c(rays_d)
    dev = ro.device
    n = ro.shape[0]
    R = int(binary.shape[0])
    b8 = binary.to(torch.uint8).contiguous()
    aabb_np = np.ascontiguousarray(aabb.detach().cpu().numpy().astype(np.float32))
    toff = None if t_offset is None else _f32c(t_offset)
    with torch.cuda.device(dev):
        scratch = torch.empty(int(_lib.lib.ngp_b200_march_scratch_bytes(n, R)), dtype=torch.uint8, device=dev)
        counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev); offsets = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        total = torch.zeros(1, dtype=torch.int64, device=dev)
        ap = C.c_void_p(aabb_np.ctypes.data)
        _lib.check(_lib.lib.ngp_b200_march_count(_P(ro), _P(rd), n, _P(b8), R, ap, float(near_plane), float(far_plane), float(dt),
                                                 _P(toff), _P(counts), _P(offsets), _P(total), _P(scratch), _stream()))
        S = int(total.item())
        ri = torch.empty(S, dtype=torch.int64, device=dev); ts = torch.empty(S, device=dev); te = torch.empty(S, device=dev)
        if S > 0:
            _lib.check(_lib.lib.ngp_b200_march_write(_P(ro), _P(rd), n, R, ap, float(near_plane), float(far_plane), float(dt),
                                                     _P(toff), _P(offsets), _P(ri), _P(ts), _P(te), _P(scratch), _stream()))
    return ri, ts, te


def _ranges(ray_indices, n_rays):
    ri = ray_indices.contiguous()
    rng = torch.empty(max(n_rays, 1), 2, dtype=torch.int32, device=ri.device)
    with torch.cuda.device(ri.device):
        _lib.check(_lib.lib.ngp_b200_ray_ranges(_P(ri), ri.numel(), n_rays, _P(rng), _stream()))
    return rng


class _Weights(torch.autograd.Function):
    @staticmethod
    def forward(ctx, t_starts, t_ends, sigmas, ranges, n_rays):
        ts, te, sg = _f32c(t_starts), _f32c(t_ends), _f32c(sigmas)
        w = torch.empty_like(sg); tr = torch.empty_like(sg); al = torch.empty_like(sg)
        with torch.cuda.device(sg.device):
            _lib.check(_lib.lib.ngp_b200_weights_fwd(_P(ts), _P(te), _P(sg), _P(ranges), n_rays, _P(w), _P(tr), _P(al), _stream()))
        ctx.save_for_backward(ts, te, sg, ranges, tr, al)
        ctx.n_rays = n_rays
        return w, tr, al

    @staticmethod
    def backward(ctx, gw, gt, ga):
        ts, te, sg, ranges, tr, al = ctx.saved_tensors
        d = torch.empty_like(sg)
        f = lambda g: None if g is None else _f32c(g)
        with torch.cuda.device(sg.device):
            _lib.check(_lib.lib.ngp_b200_weights_bwd(_P(ts), _P(te), _P(sg), _P(ranges), ctx.n_rays, _P(tr), _P(al), _P(f(gw)), _P(f(gt)),
                                                     _P(f(ga)), _P(d), _stream()))
        return None, None, d, None, None


def render_weight_from_density(t_starts, t_ends, sigmas, packed_info=None, ray_indices=None, n_rays=None, prefix_trans=None):
    """nerfacc.render_weight_from_density -> (weights, trans, alphas); packed samples, ray_indices sorted ascending."""
    if ray_indices is None or n_rays is None or prefix_trans is not None or packed_info is not None:
        raise NotImplementedError("call with ray_indices= and n_rays= (the reference's form, Instant_NGP.py:147)")
    if sigmas.numel() == 0:
        z = sigmas.new_zeros(0)
        return z, z, z
    rng = _ranges(ray_indices, int(n_rays))
    return _Weights.apply(t_starts, t_ends, sigmas, rng, int(n_rays))


class _Accumulate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weights, values, ray_indices, ranges, n_rays):
        w = _f32c(weights)
        v = None if values is None else _f32c(values)
        Cc = 1 if v is None else v.shape[-1]
        out = torch.empty(n_rays, Cc, device=w.device)
        with torch.cuda.device(w.device):
            _lib.check(_lib.lib.ngp_b200_accumulate_fwd(_P(w), _P(v), Cc, _P(ranges), n_rays, _P(out), _stream()))
        ctx.save_for_backward(w, v, ray_indices)
        ctx.Cc = Cc
        return out

    @staticmethod
    def backward(ctx, g):
        w, v, ri = ctx.saved_tensors
        g = _f32c(g)
        dw = torch.empty_like(w)
        dv = None if v is None else torch.empty_like(v)
        with torch.cuda.device(w.device):
            _lib.check(_lib.lib.ngp_b200_accumulate_bwd(_P(w), _P(v), ctx.Cc, _P(ri.contiguous()), w.numel(), _P(g), _P(dw), _P(dv), _stream()))
        return dw, dv, None, None, None


def accumulate_along_rays(weights, values=None, ray_indices=None, n_rays=None):
    """nerfacc.accumulate_along_rays: out[n_rays, C] = sum over each ray's samples of w * values (values None -> C=1)."""
    if ray_indices is None or n_rays is None:
        raise NotImplementedError("call with ray_indices= and n_rays= (the reference's form, Instant_NGP.py:148-149)")
    n_rays = int(n_rays)
    if weights.numel() == 0:
        return weights.new_zeros(n_rays, 1 if values is None else values.shape[-1])
    rng = _ranges(ray_indices, n_rays)
    return _Accumulate.apply(weights, values, ray_indices, rng, n_rays)
