"""H100-native optimisation loop around the rasterizer: the fast path for what GaussianModel +
GaussianSplatting3D.training do in the reference (MVs_Algorithms/GaussianSplatting/main_3DGS_renderer.py:236-781,
main_3DGS.py:86-232).  The reference's own Python runs unmodified over the `diff_gaussian_rasterization` shim; this
module is the packed-layout alternative: one raw-parameter buffer, fused activation, multi-view pipelined
forward/backward (gs_b200_step_device), fused chain-rule + Adam (gs_b200_adam_step), fused densification
statistics, torch-side clone/split/prune (every 100 steps).  Losses are torch ops (gs_b200.losses).
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib, camera, losses, optim_step, parallel
from .rasterizer import _ptr, _stream, knn_mean_dist2

SH_C0 = 0.28209479177387814


def expon_lr(step, lr_init, lr_final, delay_mult=1.0, max_steps=30000, delay_steps=0):
    """get_expon_lr_func (main_3DGS_renderer.py:21-43)."""
    if lr_init == lr_final:
        return lr_init
    if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
        return 0.0
    delay = delay_mult + (1 - delay_mult) * np.sin(0.5 * np.pi * np.clip(step / delay_steps, 0, 1)) if delay_steps > 0 else 1.0
    t = np.clip(step / max_steps, 0, 1)
    return float(delay * np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t))


class TrainParams:
    """GSParams defaults (main_3DGS.py:15-74)."""

    def __init__(self, **kw):
        d = dict(training_iterations=30000, batch_size=1, lambda_ssim=0.2, lambda_alpha=3.0, feature_lr=0.0025, opacity_lr=0.05,
                 scaling_lr=0.005, rotation_lr=0.001, position_lr_init=0.00016, position_lr_final=0.0000016,
                 position_lr_delay_mult=0.01, position_lr_max_steps=30000, num_pts=10000, percent_dense=0.01,
                 density_start_iter=500, density_end_iter=15000, densification_interval=100, opacity_reset_interval=3000,
                 densify_grad_threshold=0.0002, sh_degree=3, spatial_lr_scale=10.0)
        d.update(kw)
        self.__dict__.update(d)


class GaussianTrainer:
    GROUPS = ("xyz", "shs", "opacity", "scaling", "rotation")

    def __init__(self, params: TrainParams = None, device="cuda", seed=0):
        self.p = params or TrainParams()
        self.device = torch.device(device)
        self.M = (self.p.sh_degree + 1) ** 2
        self.step_count = 0
        self._init_random(self.p.num_pts, seed)

    # ---------------------------------------------------------------- packed storage
    def _sizes(self, n):
        return [3 * n, 3 * self.M * n, n, 3 * n, 4 * n]

    def _views(self, buf, n):
        out, o = {}, 0
        for name, s, shp in zip(self.GROUPS, self._sizes(n), [(n, 3), (n, self.M, 3), (n, 1), (n, 3), (n, 4)]):
            out[name] = buf[o:o + s].view(*shp); o += s
        return out

    def _alloc(self, n):
        """(Re)binds every per-Gaussian array to n rows.  Storage is grow-only: buffers are allocated for a capacity
        >= n (1.5x head room once densification starts) and the packed arrays are prefix slices of them, so a
        densification normally allocates nothing.  Two parameter sets (raw, m1, m2) exist so that the compaction kernel
        can scatter from one into the other (gs_b200_densify_apply)."""
        if n > getattr(self, "_cap", 0):
            cap = n if getattr(self, "_cap", 0) == 0 else max(n, int(1.5 * self._cap))
            ctot = sum(self._sizes(cap))
            self._store = [dict(raw=torch.zeros(ctot, device=self.device), m1=torch.zeros(ctot, device=self.device),
                                m2=torch.zeros(ctot, device=self.device)) for _ in range(2)]
            self._cur = 0
            self._aux = dict(act=torch.zeros(8 * cap, device=self.device), grads=torch.zeros(ctot + 3 * cap, device=self.device),
                             radii=torch.zeros(cap, dtype=torch.int32, device=self.device), accum=torch.zeros(cap, device=self.device),
                             denom=torch.zeros(cap, device=self.device), maxr=torch.zeros(cap, device=self.device))
            self._cap = cap
        self._bind(n, zero=True)

    def _bind(self, n, zero):
        tot = sum(self._sizes(n))
        st = self._store[self._cur]
        self.N = n
        self.raw, self.m1, self.m2 = st["raw"][:tot], st["m1"][:tot], st["m2"][:tot]
        if zero:
            self.raw.zero_(); self.m1.zero_(); self.m2.zero_()
        self.v = self._views(self.raw, n)
        self.act = self._aux["act"][:8 * n]                                     # activated opac | scales | rots
        self.a_opac, self.a_scales, self.a_rots = self.act[:n].view(n, 1), self.act[n:4 * n].view(n, 3), self.act[4 * n:].view(n, 4)
        self.grads = self._aux["grads"][:tot + 3 * n]                           # + means2D
        self.grads.zero_()
        self.g_means2D = self.grads[tot:].view(n, 3)
        self.radii = self._aux["radii"][:n]; self.radii.zero_()
        self.grad_accum, self.denom, self.max_radii2D = self._aux["accum"][:n], self._aux["denom"][:n], self._aux["maxr"][:n]
        self.grad_accum.zero_(); self.denom.zero_(); self.max_radii2D.zero_()

    def _init_random(self, n, seed):
        """initialize(None, num_pts) + create_from_pcd (main_3DGS_renderer.py:811-826, 407-433)."""
        rng = np.random.RandomState(seed)
        phis = rng.random_sample((n,)) * 2 * np.pi
        thetas = np.arccos(rng.random_sample((n,)) * 2 - 1)
        r = 0.5 * np.cbrt(rng.random_sample((n,)))
        xyz = np.stack((r * np.sin(thetas) * np.cos(phis), r * np.sin(thetas) * np.sin(phis), r * np.cos(thetas)), 1).astype(np.float32)
        col = (rng.random_sample((n, 3)) / 255.0) * SH_C0 + 0.5
        self._alloc(n)
        self.v["xyz"].copy_(torch.from_numpy(xyz))
        self.v["shs"][:, 0, :] = torch.from_numpy(((col - 0.5) / SH_C0).astype(np.float32)).to(self.device)
        d2 = torch.clamp_min(knn_mean_dist2(self.v["xyz"]), 1e-7)
        self.v["scaling"].copy_(torch.log(torch.sqrt(d2))[:, None].repeat(1, 3))
        self.v["rotation"][:, 0] = 1.0
        self.v["opacity"].fill_(math.log(0.1 / 0.9))

    # ---------------------------------------------------------------- one optimisation step
    def activate(self):
        _lib.check(_lib.lib.gs_b200_activate(self.N, _ptr(self.v["opacity"]), _ptr(self.v["scaling"]), _ptr(self.v["rotation"]),
                                             _ptr(self.a_opac), _ptr(self.a_scales), _ptr(self.a_rots), _stream()))

    def learning_rates(self, step):
        p = self.p
        lr_xyz = expon_lr(step, p.position_lr_init * p.spatial_lr_scale, p.position_lr_final * p.spatial_lr_scale,
                          p.position_lr_delay_mult, p.position_lr_max_steps)
        return np.array([lr_xyz, p.feature_lr, p.feature_lr / 20.0, p.opacity_lr, p.scaling_lr, p.rotation_lr], dtype=np.float32)

    def _cloud(self):
        cloud = optim_step.PackedParams.__new__(optim_step.PackedParams)
        cloud.means3D, cloud.shs, cloud.opacities, cloud.scales, cloud.rotations = self.v["xyz"], self.v["shs"], self.a_opac, self.a_scales, self.a_rots
        cloud.N, cloud.M, cloud.grads, cloud.radii = self.N, self.M, self.grads, self.radii
        return cloud

    def _viewset(self, views_np, W, H):
        return optim_step.ViewSet(np.ascontiguousarray(views_np, dtype=np.float32), W, H, self.p.sh_degree, self.device)

    def render_views(self, views_np, W, H, radii=None):
        """Forward only (gs_b200_render_views): images [V,5,H,W] = rgb | depth | alpha."""
        self.activate()
        imgs, _ = optim_step.render_views(self._cloud(), self._viewset(views_np, W, H), radii=radii)
        return imgs

    def forward_backward(self, views_np, W, H, loss_grad_fn):
        """ONE pipelined pass: per view forward -> loss_grad_fn(v, image, dL) -> backward; gradients wrt the activated
        parameters are summed over the views into self.grads.  Returns the images."""
        V = views_np.shape[0]
        self.activate()
        imgs = torch.empty(V, 5, H, W, device=self.device)
        dl = torch.empty(V, 5, H, W, device=self.device)
        radii = torch.empty(V, self.N, dtype=torch.int32, device=self.device)
        optim_step.step_device_loss(self._cloud(), self._viewset(views_np, W, H), loss_grad_fn, imgs, dl, radii)
        # radii of the LAST view of the batch: what the reference's densification statistics see (main_3DGS.py:211)
        self.radii.copy_(radii[V - 1])
        return imgs

    def train_step(self, views_np, W, H, ref_images, ref_masks, world=None, total_views=None, loss_fn=None):
        """ref_images [V,3,H,W], ref_masks [V,1,H,W] on device: this rank's views.  The loss terms are batch means
        (main_3DGS.py:184-192), so the loss of the global batch is the mean of per-view losses: each view's loss and
        its gradient are evaluated inside the render pipeline, between that view's forward and backward.
        Data parallel: with torch.distributed initialised (or `world` given) the packed gradient buffer is
        all-reduced once and averaged.  loss_fn=None uses the reference's loss as CUDA kernels (gs_b200_step_device_train);
        a torch callable is run per view through the host hook instead.  Returns the (global-batch) loss as a float."""
        p = self.p
        V = views_np.shape[0]
        if world is None:
            world = torch.distributed.get_world_size() if (torch.distributed.is_available() and torch.distributed.is_initialized()) else 1
        total = total_views or V * world
        per_view = torch.zeros(V, device=self.device)
        # data parallel: the all-reduce of the packed gradients is issued in Gaussian-range chunks from inside the step,
        # behind its last pass (parallel.OverlappedGradAllReduce); inactive without a process group
        ar = parallel.OverlappedGradAllReduce(self.grads, self.N, self.M, nchunks=1, enabled=world > 1)
        ar.__enter__()
        try:
            self._run_views(views_np, W, H, ref_images, ref_masks, world, total, per_view, loss_fn)
        finally:
            ar.__exit__(None, None, None)
        loss_sum = per_view.sum()
        if world > 1:
            if ar.active:
                ar.wait()
                torch.distributed.all_reduce(loss_sum)
        self._optimise(world, loss_sum)
        return float(loss_sum) / world

    def _run_views(self, views_np, W, H, ref_images, ref_masks, world, total, per_view, loss_fn):
        p = self.p
        V = views_np.shape[0]
        if loss_fn is None:
            # native path: the loss and its gradient are CUDA kernels on each view's stream (gs_loss.cu)
            self.activate()
            imgs = torch.empty(V, 5, H, W, device=self.device); dl = torch.empty(V, 5, H, W, device=self.device)
            radii = torch.empty(V, self.N, dtype=torch.int32, device=self.device)
            optim_step.step_device_train(self._cloud(), self._viewset(views_np, W, H), ref_images.contiguous(), ref_masks.contiguous(),
                                         p.lambda_ssim, p.lambda_alpha, 1.0 / total * world, imgs, dl, per_view, radii)
            self.radii.copy_(radii[V - 1])
        else:
            # any torch loss: loss_fn(images[1,3,H,W] clamped, alphas[1,1,H,W], ref[1,3,H,W], mask[1,1,H,W]) -> scalar
            def loss_grad_fn(v, img, dl):
                x = img.detach().clone().requires_grad_(True)
                loss = loss_fn(x[None, :3].clamp(0, 1), x[None, 4:5], ref_images[v:v + 1], ref_masks[v:v + 1]) * (world / total)
                loss.backward()
                dl.copy_(x.grad)
                per_view[v] = loss.detach()
            self.forward_backward(views_np, W, H, loss_grad_fn)

    def _optimise(self, world, loss_sum):
        p = self.p
        self.step_count += 1
        lrs = self.learning_rates(self.step_count - 1)
        _lib.check(_lib.lib.gs_b200_adam_step(self.N, self.M, C.c_void_p(lrs.ctypes.data), 0.9, 0.999, 1e-15, self.step_count, 1.0 / world,
                                              _ptr(self.grads), _ptr(self.raw), _ptr(self.m1), _ptr(self.m2), _stream()))
        s = self.step_count - 1
        if p.density_start_iter <= s <= p.density_end_iter:
            # NOTE: radii of the LAST view of the batch, as the reference (main_3DGS.py:211) — here also the summed means2D grad
            if world > 1:
                # the all-reduced buffer is world x the global-mean gradient (per-view loss scale world/total); Adam
                # compensates with grad_scale, the densification statistics must too or the threshold shrinks by 1/world
                self.g_means2D.mul_(1.0 / world)
            _lib.check(_lib.lib.gs_b200_densify_stats(self.N, _ptr(self.g_means2D), _ptr(self.radii), _ptr(self.grad_accum),
                                                      _ptr(self.denom), _ptr(self.max_radii2D), _stream()))
            if s % p.densification_interval == 0:
                if world > 1:
                    parallel.allreduce_densify_stats(self.grad_accum, self.denom, self.max_radii2D)
                self.densify_and_prune(p.densify_grad_threshold, 0.005, 4.0, 1.0)
            if s % p.opacity_reset_interval == 0:
                self.reset_opacity()

    # ---------------------------------------------------------------- densification (torch-side, infrequent)
    def _rebuild(self, keep_idx, new):
        """keep rows `keep_idx` of every group (+Adam moments), append `new` rows (zero moments)."""
        old_v, old_m1, old_m2, n_old = self.v, self._views(self.m1, self.N), self._views(self.m2, self.N), self.N
        n_new = keep_idx.numel() + (new["xyz"].shape[0] if new else 0)
        raws = {k: old_v[k][keep_idx] for k in self.GROUPS}
        m1s = {k: old_m1[k][keep_idx] for k in self.GROUPS}; m2s = {k: old_m2[k][keep_idx] for k in self.GROUPS}
        self._alloc(n_new)
        nm1, nm2 = self._views(self.m1, n_new), self._views(self.m2, n_new)
        k0 = keep_idx.numel()
        for k in self.GROUPS:
            self.v[k][:k0] = raws[k]; nm1[k][:k0] = m1s[k]; nm2[k][:k0] = m2s[k]
            if new:
                self.v[k][k0:] = new[k]

    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, generator=None, normal_samples=None):
        """densify_by_clone_and_split + prune (main_3DGS_renderer.py:641-668, 752-781).
        CUDA tensors: stream compaction kernels over the packed buffers (gs_b200_densify_plan / _apply): no boolean-mask
        indexing, no re-allocation below the capacity, one 40-byte host read for the counts.  `normal_samples`
        ([2 x split parents, 3] standard normal) replaces the draw of densify_and_split (:653) for replay tests.
        CPU tensors (fixture tests of the host logic): the torch restatement below."""
        if self.raw.is_cuda:
            return self._densify_and_prune_cuda(max_grad, min_opacity, extent, generator, normal_samples)
        return self._densify_and_prune_torch(max_grad, min_opacity, extent, max_screen_size, generator)

    def _densify_and_prune_cuda(self, max_grad, min_opacity, extent, generator, normal_samples):
        p, N, dev = self.p, self.N, self.device
        with torch.cuda.device(dev):
            work, counts, scratch, zbuf = self._densify_workspace()
            _lib.check(_lib.lib.gs_b200_densify_plan(N, _ptr(self.v["opacity"]), _ptr(self.v["scaling"]), _ptr(self.grad_accum), _ptr(self.denom),
                                                     float(max_grad), float(min_opacity), float(extent), float(p.percent_dense),
                                                     _ptr(work), _ptr(counts), _ptr(scratch), _stream()))
            n_keep, n_clone, n_sp, n_spk, clone_total = (int(x) for x in counts.cpu())          # the one host sync
            n_new = n_keep + n_clone + 2 * n_spk
            if normal_samples is None:
                z = zbuf[:6 * n_sp].view(2 * n_sp, 3).normal_(generator=generator)      # (n_sp <= N <= capacity)
            else:
                z = normal_samples.to(dev).float().contiguous()
                assert z.shape == (2 * n_sp, 3), (z.shape, n_sp)
            src = self._store[self._cur]
            src_views = (src["raw"][:self.raw.numel()], src["m1"][:self.raw.numel()], src["m2"][:self.raw.numel()])
            if n_new > self._cap:                # grow-only: both sets move to the new capacity, the live one keeps its contents
                old_n = self.N
                self._alloc_grow(n_new)
                src = self._store[self._cur]
                tot_old = sum(self._sizes(old_n))
                src_views = (src["raw"][:tot_old], src["m1"][:tot_old], src["m2"][:tot_old])
            dst = self._store[1 - self._cur]
            tot_new = sum(self._sizes(n_new))
            if n_new > 0:
                _lib.check(_lib.lib.gs_b200_densify_apply(N, self.M, _ptr(src_views[0]), _ptr(src_views[1]), _ptr(src_views[2]), _ptr(work),
                                                          n_keep, n_clone, n_sp, n_spk, _ptr(z) if n_sp else None,
                                                          _ptr(dst["raw"][:max(tot_new, 1)]), _ptr(dst["m1"][:max(tot_new, 1)]),
                                                          _ptr(dst["m2"][:max(tot_new, 1)]), _stream()))
            self._cur = 1 - self._cur
            self._bind(n_new, zero=False)
        return dict(cloned=clone_total, split=n_sp, pruned=N - n_keep, n=self.N, n_before=N)

    def _densify_workspace(self):
        """Plan arrays of the densification kernels, sized for the capacity and kept with it (grow-only like the rest):
        a densification that fits the capacity performs no device allocation at all."""
        ws = getattr(self, "_dws", None)
        if ws is None or ws["cap"] < self._cap:
            cap = self._cap
            ws = dict(cap=cap, work=torch.empty(8 * cap, dtype=torch.int32, device=self.device),
                      counts=torch.empty(5, dtype=torch.int64, device=self.device),
                      scratch=torch.empty(int(_lib.lib.gs_b200_densify_scratch_bytes(cap)), dtype=torch.uint8, device=self.device),
                      z=torch.empty(6 * cap, device=self.device))               # children offsets: 2 x split parents x 3 normals
            self._dws = ws
        return ws["work"], ws["counts"], ws["scratch"], ws["z"]

    def _alloc_grow(self, n):
        """capacity growth that keeps the live parameter set (used when a densification outgrows the buffers)."""
        cap = max(n, int(1.5 * self._cap))
        ctot = sum(self._sizes(cap))
        old = self._store
        self._store = [dict(raw=torch.zeros(ctot, device=self.device), m1=torch.zeros(ctot, device=self.device),
                            m2=torch.zeros(ctot, device=self.device)) for _ in range(2)]
        for k in ("raw", "m1", "m2"):
            self._store[self._cur][k][:old[self._cur][k].numel()].copy_(old[self._cur][k])
        self._aux = dict(act=torch.zeros(8 * cap, device=self.device), grads=torch.zeros(ctot + 3 * cap, device=self.device),
                         radii=torch.zeros(cap, dtype=torch.int32, device=self.device), accum=torch.zeros(cap, device=self.device),
                         denom=torch.zeros(cap, device=self.device), maxr=torch.zeros(cap, device=self.device))
        self._cap = cap

    def _densify_and_prune_torch(self, max_grad, min_opacity, extent, max_screen_size, generator=None):
        """The same rules as torch tensor surgery (the host-logic restatement the CPU fixture test pins to the reference)."""
        p = self.p
        grads = self.grad_accum / self.denom
        grads[grads.isnan()] = 0.0
        scal = torch.exp(self.v["scaling"]).max(dim=1).values
        big = scal > p.percent_dense * extent
        clone = (grads >= max_grad) & ~big
        split = (grads >= max_grad) & big                       # evaluated on the pre-clone set: clones carry zero grad
        idx_c = torch.nonzero(clone)[:, 0]; idx_s = torch.nonzero(split)[:, 0]
        new = {k: self.v[k][idx_c].clone() for k in self.GROUPS}
        if idx_s.numel():
            Nn = 2
            stds = torch.exp(self.v["scaling"][idx_s]).repeat(Nn, 1)
            samples = torch.normal(torch.zeros_like(stds), stds, generator=generator)
            q = self.v["rotation"][idx_s]
            q = q / q.norm(dim=1, keepdim=True)
            r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
            R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y), 2 * (x * y + r * z), 1 - 2 * (x * x + z * z),
                             2 * (y * z - r * x), 2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=1).view(-1, 3, 3).repeat(Nn, 1, 1)
            sp = {"xyz": torch.bmm(R, samples.unsqueeze(-1)).squeeze(-1) + self.v["xyz"][idx_s].repeat(Nn, 1),
                  "scaling": torch.log(torch.exp(self.v["scaling"][idx_s]).repeat(Nn, 1) / (0.8 * Nn)),
                  "rotation": self.v["rotation"][idx_s].repeat(Nn, 1), "shs": self.v["shs"][idx_s].repeat(Nn, 1, 1),
                  "opacity": self.v["opacity"][idx_s].repeat(Nn, 1)}
            new = {k: torch.cat([new[k], sp[k]], dim=0) for k in self.GROUPS}
        # prune: split parents, low opacity, big in world space.  The reference's screen-size rule
        # (`max_radii2D > max_screen_size`, :774) never fires as written: densification_postfix has already reset
        # max_radii2D to zeros for every point (:636-639) by the time prune() reads it — reproduced here (pinned by
        # tests/test_golden_training.py against the reference's own class).
        n_old = self.N
        opac = torch.sigmoid(self.v["opacity"]).squeeze(1)
        prune_old = split | (opac < min_opacity) | (scal > 0.1 * extent)
        n_op = torch.sigmoid(new["opacity"]).squeeze(1); n_sc = torch.exp(new["scaling"]).max(dim=1).values
        keep_new = ~((n_op < min_opacity) | (n_sc > 0.1 * extent))
        new = {k: v[keep_new] for k, v in new.items()}
        self._rebuild(torch.nonzero(~prune_old)[:, 0], new)
        return dict(cloned=int(idx_c.numel()), split=int(idx_s.numel()), pruned=int(prune_old.sum()), n=self.N, n_before=n_old)

    def reset_opacity(self):
        o = torch.sigmoid(self.v["opacity"])
        o = torch.minimum(o, torch.full_like(o, 0.01))
        self.v["opacity"].copy_(torch.log(o / (1 - o)))
        self._views(self.m1, self.N)["opacity"].zero_(); self._views(self.m2, self.N)["opacity"].zero_()
