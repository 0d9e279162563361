"""CPU oracle for the Instant-NGP path (hash-grid encode + occupancy-grid ray march + volume composite)
— TEST INFRASTRUCTURE ONLY.

    PARITY UNPINNED: kiui 0.2.14 (`kiui.gridencoder`, torch-ngp's grid encoder; my-reqs.txt:50) and nerfacc
    0.5.3 (my-reqs.txt:69) are un-vendored third-party packages, absent from the reference source tree and not
    installable offline; the reference has no tests or golden vectors for them (SURVEY.md §4, §8c).

Restates the published algorithms (Müller et al. 2022 multiresolution hash encoding as implemented by
torch-ngp; Li et al. 2023 nerfacc occupancy-grid sampling and packed volume rendering; SURVEY.md App. A.3-A.4)
for what the reference calls at MVs_Algorithms/NeRF/Instant_NGP.py:

  GridEncoder(num_levels=12)(xs), .grad_total_variation(w)          :22,32-33,73,80,195
  OccGridEstimator(roi_aabb, resolution=64, levels=1)               :30
      .update_every_n_steps / .sampling                             :117,129-138
  render_weight_from_density, accumulate_along_rays                 :147-149
  kiui.nn.MLP, trunc_exp; get_rays                                  :34-35,37-70,82

Arithmetic contract (bit-exact integer outputs against the CUDA path): hash-grid corner indices and the
packed sample list (ray_indices, t_starts, t_ends) are produced with the exact fp32 operation order below
(no FMA), so they compare bit-for-bit; encoded features, weights and gradients compare with tolerances.

Marching rule restated here (fixed-step marching with empty-space skipping): along each ray, with
t_enter = max(near, aabb entry) (+ U[0,1)*dt when stratified) and t_exit = min(far, aabb exit), the candidate
intervals are [t_enter + k*dt, t_enter + (k+1)*dt), k = 0,1,...; an interval becomes a sample iff its midpoint is
before t_exit and falls in an occupied cell of the binary grid.  Samples are then pruned by the transmittance
test T >= early_stop_eps evaluated with the current densities (render_visibility_from_density).
"""
from __future__ import annotations

import math

import numpy as np
import torch

PRIMES = (1, 2654435761, 805459861)


# --------------------------------------------------------------------------------------------------
# hash grid (torch-ngp / kiui.gridencoder)
# --------------------------------------------------------------------------------------------------
def grid_offsets(num_levels=16, level_dim=2, per_level_scale=2.0, base_resolution=16, log2_hashmap_size=19,
                 input_dim=3, align_corners=False):
    max_params = 2 ** log2_hashmap_size
    offsets, off = [], 0
    for i in range(num_levels):
        res = int(np.ceil(base_resolution * per_level_scale ** i))
        n = min(max_params, (res if align_corners else res + 1) ** input_dim)
        n = int(np.ceil(n / 8) * 8)
        offsets.append(off); off += n
    offsets.append(off)
    return np.array(offsets, dtype=np.int64)


def _level_geometry(level, per_level_scale, base_resolution):
    S = np.float32(np.log2(per_level_scale))
    scale = np.float32(np.exp2(np.float32(level) * S) * np.float32(base_resolution) - np.float32(1.0))
    resolution = int(np.ceil(scale)) + 1
    return scale, resolution


def grid_corner_indices(x01: torch.Tensor, level: int, offsets, per_level_scale=2.0, base_resolution=16):
    """x01 [N,3] in [0,1] (fp32). Returns (idx [N,8] int64 into this level's table, w [N,8], frac [N,3])."""
    scale, res = _level_geometry(level, per_level_scale, base_resolution)
    hsize = int(offsets[level + 1] - offsets[level])
    pos = x01 * float(scale) + 0.5
    pg = torch.floor(pos)
    frac = pos - pg
    pg = pg.to(torch.int64)
    idxs, ws = [], []
    stride_full = (res + 1) ** 3
    for c in range(8):
        bits = [(c >> d) & 1 for d in range(3)]
        g = [pg[:, d] + bits[d] for d in range(3)]
        w = torch.ones_like(frac[:, 0])
        for d in range(3):
            w = w * (frac[:, d] if bits[d] else (1.0 - frac[:, d]))
        if stride_full <= hsize:        # dense level
            idx = g[0] + g[1] * (res + 1) + g[2] * (res + 1) * (res + 1)
        else:
            idx = torch.zeros_like(g[0])
            for d in range(3):
                idx = idx ^ ((g[d] * PRIMES[d]) & 0xFFFFFFFF)
        idxs.append(idx % hsize); ws.append(w)
    return torch.stack(idxs, 1), torch.stack(ws, 1), frac


def grid_encode(x: torch.Tensor, embeddings: torch.Tensor, offsets, bound=1.0, num_levels=16, level_dim=2,
                per_level_scale=2.0, base_resolution=16):
    """x [N,3] in [-bound,bound] -> [N, L*C]; differentiable wrt embeddings."""
    x01 = (x.to(torch.float32) + bound) / (2 * bound)
    outs = []
    for l in range(num_levels):
        idx, w, _ = grid_corner_indices(x01, l, offsets, per_level_scale, base_resolution)
        table = embeddings[int(offsets[l]):int(offsets[l + 1])]
        feat = (table[idx] * w[:, :, None].to(embeddings.dtype)).sum(dim=1)         # [N,C]
        outs.append(feat)
    return torch.cat(outs, dim=1)


def grad_total_variation(x: torch.Tensor, embeddings: torch.Tensor, offsets, weight, bound=1.0, num_levels=16,
                         per_level_scale=2.0, base_resolution=16):
    """Gradient of the L1 total-variation regulariser at the cells containing the sample points, as ADDED to
    embeddings.grad by GridEncoder.grad_total_variation: for the cell's base corner c and each axis, weight *
    (sign(c - right) + sign(c - left)) with neighbours inside [0,res]."""
    x01 = (x.to(torch.float32) + bound) / (2 * bound)
    g = torch.zeros_like(embeddings)
    for l in range(num_levels):
        scale, res = _level_geometry(l, per_level_scale, base_resolution)
        hsize = int(offsets[l + 1] - offsets[l])
        pg = torch.floor(x01 * float(scale) + 0.5).to(torch.int64)

        def index(gx, gy, gz):
            if (res + 1) ** 3 <= hsize:
                return (gx + gy * (res + 1) + gz * (res + 1) * (res + 1)) % hsize
            return (((gx * PRIMES[0]) & 0xFFFFFFFF) ^ ((gy * PRIMES[1]) & 0xFFFFFFFF) ^ ((gz * PRIMES[2]) & 0xFFFFFFFF)) % hsize
        table = embeddings[int(offsets[l]):int(offsets[l + 1])]
        ci = index(pg[:, 0], pg[:, 1], pg[:, 2])
        cur = table[ci]
        acc = torch.zeros_like(cur)
        for d in range(3):
            for s in (+1, -1):
                q = pg.clone(); q[:, d] += s
                ok = (q[:, d] >= 0) & (q[:, d] <= res)
                nb = table[index(q[:, 0].clamp(0, res), q[:, 1].clamp(0, res), q[:, 2].clamp(0, res))]
                acc = acc + torch.where(ok[:, None], torch.sign(cur - nb), torch.zeros_like(cur))
        g[int(offsets[l]):int(offsets[l + 1])].index_add_(0, ci, weight * acc)
    return g


# --------------------------------------------------------------------------------------------------
# rays, occupancy grid, marching (nerfacc)
# --------------------------------------------------------------------------------------------------
def get_rays(pose: np.ndarray, h: int, w: int, fovy_deg: float):
    """InstantNGP.get_rays (Instant_NGP.py:37-70), OpenGL convention, pixel centres at +0.5."""
    pose = torch.from_numpy(np.asarray(pose, dtype=np.float32))
    x, y = torch.meshgrid(torch.arange(w), torch.arange(h), indexing="xy")
    x = x.flatten(); y = y.flatten()
    cx, cy = w * 0.5, h * 0.5
    focal = h * 0.5 / np.tan(0.5 * np.deg2rad(fovy_deg))
    dirs = torch.nn.functional.pad(torch.stack([(x - cx + 0.5) / focal, (y - cy + 0.5) / focal * -1.0], dim=-1), (0, 1), value=-1.0)
    rays_d = dirs.float() @ pose[:3, :3].transpose(0, 1)
    rays_o = pose[:3, 3].unsqueeze(0).expand_as(rays_d)
    rays_d = rays_d / torch.sqrt(torch.clamp((rays_d * rays_d).sum(-1, keepdim=True), min=1e-20))
    return rays_o.contiguous(), rays_d.contiguous()


def ray_aabb(rays_o, rays_d, aabb):
    """Slab test in fp32, explicit op order: t = (plane - o) * (1/d)."""
    lo, hi = aabb[:3], aabb[3:]
    inv = 1.0 / rays_d
    t0 = (lo[None] - rays_o) * inv
    t1 = (hi[None] - rays_o) * inv
    tmin = torch.minimum(t0, t1).max(dim=1).values
    tmax = torch.maximum(t0, t1).min(dim=1).values
    return tmin, tmax


def march(rays_o, rays_d, binary: torch.Tensor, aabb: torch.Tensor, near, far, dt, t_offset=None):
    """Packed samples (ray_indices int64, t_starts, t_ends) per the marching rule in the module docstring.
    binary: [R,R,R] bool indexed [x,y,z]; t_offset: optional per-ray stratified offset in [0,dt)."""
    R = binary.shape[0]
    n = rays_o.shape[0]
    f32 = torch.float32
    tmin, tmax = ray_aabb(rays_o.to(f32), rays_d.to(f32), aabb.to(f32))
    t_enter = torch.maximum(tmin, torch.full_like(tmin, near))
    t_exit = torch.minimum(tmax, torch.full_like(tmax, far))
    if t_offset is not None:
        t_enter = t_enter + t_offset
    hit = t_exit > t_enter
    dtf = torch.tensor(dt, dtype=f32)
    span = torch.where(hit, t_exit - t_enter, torch.zeros_like(t_exit))     # NaN for rays in a face plane (no hit)
    kmax = int(math.ceil(float(span.max()) / dt)) + 1 if n else 0
    k = torch.arange(kmax, dtype=f32, device=rays_o.device)[None, :]     # (runs on CUDA tensors too: same fp32 ops)
    ts = t_enter[:, None] + k * dtf
    te = t_enter[:, None] + (k + 1.0) * dtf
    tm = (ts + te) * 0.5
    valid = hit[:, None] & (tm < t_exit[:, None])
    p = rays_o[:, None, :] + rays_d[:, None, :] * tm[:, :, None]
    lo, hi = aabb[:3].to(f32), aabb[3:].to(f32)
    cell = torch.floor((p - lo) / (hi - lo) * float(R)).to(torch.int64)
    inb = ((cell >= 0) & (cell < R)).all(dim=-1)
    cc = cell.clamp(0, R - 1)
    occ = binary[cc[..., 0], cc[..., 1], cc[..., 2]]
    keep = valid & inb & occ
    ri, ki = torch.nonzero(keep, as_tuple=True)
    return ri.to(torch.int64), ts[ri, ki].contiguous(), te[ri, ki].contiguous()


def packed_ranges(ray_indices: torch.Tensor, n_rays: int):
    cnt = torch.bincount(ray_indices, minlength=n_rays)
    start = torch.cumsum(cnt, 0) - cnt
    return start, cnt


def render_weight_from_density(t_starts, t_ends, sigmas, ray_indices, n_rays):
    """alpha = 1-exp(-sigma*dt); T = exclusive cumprod(1-alpha) per ray; w = T*alpha. Differentiable wrt sigmas."""
    alphas = 1.0 - torch.exp(-sigmas * (t_ends - t_starts))
    # exclusive cumprod per segment via log-space-free sequential scan (small cases) — exact recurrence
    start, cnt = packed_ranges(ray_indices, n_rays)
    trans = torch.ones_like(alphas)
    one_m = 1.0 - alphas
    # vectorised segmented exclusive cumprod: cumprod over the whole array divided by the segment start product
    # is numerically fragile; do it per segment for the oracle
    out = []
    for s, c in zip(start.tolist(), cnt.tolist()):
        if c == 0:
            continue
        seg = one_m[s:s + c]
        cp = torch.cumprod(seg, 0)
        out.append(torch.cat([torch.ones(1, dtype=seg.dtype), cp[:-1]]))
    trans = torch.cat(out) if out else trans
    return trans * alphas, trans, alphas


def visibility_mask(t_starts, t_ends, sigmas, ray_indices, n_rays, early_stop_eps=1e-4, alpha_thre=0.0):
    w, trans, alphas = render_weight_from_density(t_starts, t_ends, sigmas, ray_indices, n_rays)
    return (trans >= early_stop_eps) & (alphas >= alpha_thre)


def accumulate_along_rays(weights, values, ray_indices, n_rays):
    if values is None:
        src = weights[:, None]
    else:
        src = weights[:, None] * values
    out = torch.zeros(n_rays, src.shape[1], dtype=src.dtype)
    return out.index_add(0, ray_indices, src)


def trunc_exp(x):
    """kiui.nn.trunc_exp: exp forward, backward g*exp(clamp(x, max=15))."""
    class _F(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x):
            ctx.save_for_backward(x)
            return torch.exp(x)

        @staticmethod
        def backward(ctx, g):
            (x,) = ctx.saved_tensors
            return g * torch.exp(x.clamp(max=15))
    return _F.apply(x)
