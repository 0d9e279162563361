"""FlexiCubes on the H100 (csrc/ngp_flexicubes.cu via gs_b200.isosurface.FlexiCubes): every fixture case of the
reference (tests/golden/ref_flexicubes.npz) and the trainer-scale grids against the float64 torch oracle
(oracle/fc_oracle.py) on the device, in faces (exactly), vertices, L_dev and the gradients to x, s, beta, alpha and
gamma; run-to-run bit identity; the current stream; host reads and launches; error paths; and the FlexiCubes node's
step (extraction -> nvdiffrast shim render -> loss) against the same step with the oracle extraction."""
import os
import warnings

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import fc_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
Z = np.load(os.path.join(GOLDEN, "ref_flexicubes.npz"))


def _fc(ws=0.99):
    from gs_b200.isosurface import FlexiCubes
    return FlexiCubes(device=DEV, weight_scale=ws)


def _cuda_fn(fc, res, training):
    _, cubes = fc.construct_voxel_grid(res)
    return lambda x, s, b, a, g: fc(x, s, cubes, res, beta_fx12=b, alpha_fx8=a, gamma_f=g, training=training)


def _oracle_fn(res, training, ws, dtype=torch.float64):
    return lambda x, s, b, a, g: O.flexicubes(x, s, res, b, a, g, training=training, weight_scale=ws, dtype=dtype)


def _close(a, b, atol, what):
    err = float((a.double() - b.double()).abs().max()) if a.numel() else 0.0
    assert err <= atol, (what, err)


def _grads_close(ga, gb, rtol, what):
    for k in ("gx", "gs", "gw"):
        if gb.get(k) is None:
            assert ga.get(k) is None, (what, k)
            continue
        scale = float(gb[k].abs().max())
        err = float((ga[k].double() - gb[k].double()).abs().max())
        assert err <= rtol * max(scale, 1e-12), (what, k, err, scale)


# Fixture cases with s == 0 exactly at some grid points: there a group's |d_e - mean(d)| can sit at its kink, and
# which subgradient fp arithmetic picks depends on the last bits.  The fp32 oracle restatement on the same device
# differs from the fp64 one there by as much as the kernels do (up to ~1e-3 of the largest gradient), so those cases
# are held to 1e-3; every other case to 1e-4.
KINK_CASES = {"zeros": 1e-3, "boundary": 1e-3}


def _run_both(res, x, s, w, given, training, ws, z=Z, grtol=1e-4):
    """CUDA and the fp64 oracle on the same inputs: the outputs come in the same order, so faces compare exactly."""
    v, f, L, _, g = O.run_with_grads(_cuda_fn(_fc(ws), res, training), x, s, w, given, z)
    ov, of, oL, (keys,), og = O.run_with_grads(_oracle_fn(res, training, ws), x, s, w, given, z)
    assert v.dtype == torch.float32 and f.dtype == torch.int64 and L.dtype == torch.float32
    assert v.device == DEV and f.device == DEV and L.device == DEV
    assert v.shape == ov.shape and f.shape == of.shape and L.shape == oL.shape, (v.shape, ov.shape, f.shape, of.shape)
    assert torch.equal(f, of)
    _close(v, ov, 1e-5, "verts")
    _close(L, oL, 1e-5, "L_dev")
    if og is not None:
        _grads_close(g, og, grtol, "grads")
    return v, f, L, keys, g


@pytest.mark.parametrize("name", ["sphere", "random", "boundary", "zeros", "inside", "outside"])
def test_fixture_cases_match_the_reference_and_the_oracle(name):
    res, x, s, w = O.fixture_inputs(Z, name, DEV)
    for ws, given, training in O.VARIANTS:
        tag = f"{name}/{ws}/{given}/{training}"
        grtol = KINK_CASES.get(name, 1e-4)
        v, f, L, keys, g = _run_both(res, x, s, w, given, bool(training), ws, grtol=grtol)
        O.assert_matches_fixture(Z, tag, v, f, L, keys, g, grtol=grtol)


def _trainer_inputs(res, seed):
    """FlexiCubesTrainer.__init__ / training (flexicubes_trainer.py:48-56, 133): grid x2, SDF rand - 0.1, zero
    weights, and a random deform through tanh."""
    fc = _fc()
    x, _ = fc.construct_voxel_grid(res)
    x *= 2
    g = torch.Generator(device=DEV).manual_seed(seed)
    sdf = torch.rand(x.shape[0], generator=g, device=DEV) - 0.1
    deform = torch.randn(x.shape, generator=g, device=DEV)
    r = res if isinstance(res, int) else max(res)
    xd = x + (2 - 1e-8) / (r * 2) * torch.tanh(deform)
    F = res ** 3 if isinstance(res, int) else res[0] * res[1] * res[2]
    w = torch.zeros((F, 21), device=DEV)
    return xd, sdf, w


@pytest.mark.parametrize("res", [128, (96, 128, 64)])
@pytest.mark.parametrize("training", [True, False])
def test_trainer_scale_matches_the_oracle(res, training):
    x, s, w = _trainer_inputs(res, seed=5)
    _run_both(res, x, s, w, 1, training, 0.99)


def test_trainer_scale_with_random_weights_matches_the_oracle():
    x, s, _ = _trainer_inputs(64, seed=6)
    w = torch.randn((64 ** 3, 21), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV)
    for training in (True, False):
        _run_both(64, x, s, w, 1, training, 0.99)


def _bits(t):
    return t.detach().contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def test_two_runs_are_bit_identical():
    x, s, w = _trainer_inputs(96, seed=8)
    w = w + 0.3 * torch.randn(w.shape, generator=torch.Generator(device=DEV).manual_seed(9), device=DEV)
    runs = []
    for _ in range(2):
        v, f, L, _, g = O.run_with_grads(_cuda_fn(_fc(), 96, True), x, s, w, 1, Z)
        runs.append([v, f, L, g["gx"], g["gs"], g["gw"]])
    for a, b in zip(*runs):
        assert torch.equal(_bits(a), _bits(b))


def test_runs_on_the_current_stream():
    x, s, w = _trainer_inputs(48, seed=10)
    ref = O.run_with_grads(_cuda_fn(_fc(), 48, True), x, s, w, 1, Z)
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)              # keeps the side stream busy: work on another stream would race
        got = O.run_with_grads(_cuda_fn(_fc(), 48, True), x, s, w, 1, Z)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for a, b in zip(ref[:3], got[:3]):
        assert torch.equal(_bits(a), _bits(b))
    for k in ("gx", "gs", "gw"):
        assert torch.equal(_bits(ref[4][k]), _bits(got[4][k]))


def test_one_host_read_per_forward_and_none_in_the_backward():
    from gs_b200 import _lib
    fc = _fc()
    res = 64
    _, cubes = fc.construct_voxel_grid(res)
    x, s, w = _trainer_inputs(res, seed=11)
    s = s.clone().requires_grad_(True)
    wp = w.clone().requires_grad_(True)
    call = lambda: fc(x, s, cubes, res, beta_fx12=wp[:, :12], alpha_fx8=wp[:, 12:20], gamma_f=wp[:, 20],
                      training=True)
    call()                                         # recognises cube_fx8 (a one-time check)
    torch.cuda.synchronize()
    n0 = _lib.lib.gs_b200_launch_count()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            v, f, L = call()
        n1 = _lib.lib.gs_b200_launch_count()
        loss = v.square().sum() + L.mean()
        torch.cuda.set_sync_debug_mode("error")
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    n2 = _lib.lib.gs_b200_launch_count()
    syncs = [r for r in rec if "synchroniz" in str(r.message)]
    assert len(syncs) == 1, [str(r.message) for r in syncs]
    assert n2 - n1 == 3                            # quad partials, per-cube gradients, per-point gather
    assert n1 - n0 >= 3
    print("launches: forward", n1 - n0, "backward", n2 - n1)


def test_error_paths():
    fc = _fc()
    x, cubes = fc.construct_voxel_grid(8)
    s = x.norm(dim=-1) - 0.3
    with pytest.raises(ValueError):
        fc(x, s, cubes.flip(0).contiguous(), 8)
    with pytest.raises(ValueError):
        fc(x, s, cubes, 9)
    with pytest.raises(NotImplementedError):
        fc(x, s, cubes, 8, output_tetmesh=True)
    with pytest.raises(NotImplementedError):
        fc(x, s, cubes, 8, grad_func=lambda p: p)
    with pytest.raises(TypeError):
        fc(x.cpu(), s.cpu(), cubes.cpu(), 8)
    v, f, L = fc(x, s, cubes, 8)
    assert v.shape[0] > 0 and f.shape[1] == 3
    c2 = cubes.clone()
    fc(x, s, c2, 8)
    c2[0, 0] = 5                                   # an in-place edit is seen through the version counter
    with pytest.raises(ValueError):
        fc(x, s, c2, 8)


def test_empty_surface_returns_the_reference_shapes():
    fc = _fc()
    x, cubes = fc.construct_voxel_grid(6)
    for sv in (1.0, -1.0):
        s = torch.full((x.shape[0],), sv, device=DEV, requires_grad=True)
        v, f, L = fc(x, s, cubes, 6, training=True)
        assert v.shape == (0, 3) and f.shape == (0, 3) and L.shape == (0,) and f.dtype == torch.int64
        (v.sum() + L.sum()).backward()
        assert s.grad is not None and not s.grad.any()


def _render_loss(dr, v, f, mv, mvp, res, tmask, tdepth, L, weight):
    """FlexiCubesRenderer.render_mesh (mask + depth) and the trainer's loss (flexicubes_trainer.py:139-155, without
    the SDF regulariser, which does not touch the extraction)."""
    hom = torch.nn.functional.pad(v[None], (0, 1), value=1.0)
    pos = torch.matmul(hom, mvp.transpose(1, 2))
    fi = f.int()
    rast, _ = dr.rasterize(dr.RasterizeCudaContext(), pos, fi, res)
    a_idx = rast[..., -1:] > 0
    alpha = a_idx.float()
    mask = dr.antialias(alpha, rast, pos, fi)
    v_cam = torch.matmul(hom, mv.transpose(1, 2))
    depth, _ = dr.interpolate(v_cam[..., [2]].contiguous(), rast, fi)
    dm = torch.clamp(depth[a_idx], min=-5.5, max=-0.5)
    depth = depth.clone()
    depth[a_idx] = (dm + 5.5) / 5.0
    depth[~a_idx] = 0
    mask_loss = (mask - tmask).abs().mean()
    depth_loss = ((((depth - tdepth) * tmask) ** 2).sum(-1) + 1e-8).sqrt().mean() * 100.0
    return mask_loss + depth_loss + L.mean() * 0.5 + weight[:, :20].abs().mean() * 0.1


def test_trainer_step_gradients_match_the_oracle_extraction():
    import nvdiffrast.torch as dr
    from oracle import dr_oracle as D
    from oracle import gs_oracle as G
    res = 32
    fc = _fc()
    x0, cubes = fc.construct_voxel_grid(res)
    x0 *= 2
    gen = torch.Generator(device=DEV).manual_seed(12)
    sdf0 = x0.norm(dim=-1) - 0.7 + 0.05 * torch.randn(x0.shape[0], generator=gen, device=DEV)
    deform0 = 0.5 * torch.randn(x0.shape, generator=gen, device=DEV)
    weight0 = 0.3 * torch.randn((res ** 3, 21), generator=gen, device=DEV)
    H = W = 96
    proj = torch.from_numpy(D.gl_perspective(45.0, 1.0).astype(np.float32)).to(DEV)
    poses = [G.orbit_camera(el, az, 3.0) for el, az in ((10, 0), (-20, 90), (30, 200), (0, 300))]
    mv = torch.stack([torch.inverse(torch.from_numpy(p)) for p in poses]).to(DEV)
    mvp = torch.matmul(proj[None], mv)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, H, device=DEV), torch.linspace(-1, 1, W, device=DEV), indexing="ij")
    tmask = ((xx ** 2 + yy ** 2) < 0.3).float()[None, ..., None].expand(4, H, W, 1).contiguous()
    tdepth = tmask * 0.45

    snap = {}

    def step(extract):
        sdf = sdf0.clone().requires_grad_(True)
        deform = deform0.clone().requires_grad_(True)
        weight = weight0.clone().requires_grad_(True)
        grid = x0 + (2 - 1e-8) / (res * 2) * torch.tanh(deform)
        v, f, L = extract(grid, sdf, weight)[:3]
        # the renderer sees the same vertex bits in both pipelines (the extractions agree to ~1e-7, but a silhouette
        # pixel flipped by that would change the rasteriser's gradients), so what is compared is the extraction's
        # backward under the same upstream gradients
        if snap:
            v = v + (snap["v"] - v).detach()
            L = L + (snap["L"] - L).detach()
        else:
            snap.update(v=v.detach(), L=L.detach())
        loss = _render_loss(dr, v, f, mv, mvp, (H, W), tmask, tdepth, L, weight)
        loss.backward()
        return float(loss.detach()), sdf.grad, deform.grad, weight.grad, f.shape[0]

    cuda = step(lambda g, s, w: fc(g, s, cubes, res, beta_fx12=w[:, :12], alpha_fx8=w[:, 12:20], gamma_f=w[:, 20],
                                   training=True))
    orc = step(lambda g, s, w: O.flexicubes(g, s, res, w[:, :12], w[:, 12:20], w[:, 20], training=True,
                                            weight_scale=0.99, dtype=torch.float32))
    assert cuda[4] == orc[4] and cuda[4] > 1000
    assert abs(cuda[0] - orc[0]) <= 1e-4 * abs(orc[0])
    for a, b, n in zip(cuda[1:4], orc[1:4], ("sdf", "deform", "weight")):
        rel = float((a - b).double().norm() / (b.double().norm() + 1e-30))
        assert float(b.abs().max()) > 0 and rel < 1e-3, (n, rel)
