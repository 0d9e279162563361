"""The pipelined step (gs_b200_step_device) zeroes each view's SplatGrad slice on that view's stream.  A view that
renders no (tile, splat) pair has no composite backward, but the batched preprocess-backward still reads its slice for
every Gaussian with radii > 0 in it, so that slice must be zeroed too -- or the previous step's sums leak into the
gradients."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
N, W, H, DEG = 20_000, 320, 240, 0
DEAD_OPACITY = 0.002          # below 1/255: such a splat is listed in no tile and blended into no pixel


def _ball(g, n, r):
    v = torch.randn(n, 3, generator=g)
    return torch.nn.functional.normalize(v, dim=1) * r * torch.rand(n, 1, generator=g) ** (1 / 3)


def make_case(dev):
    """Two orbit views facing each other across the origin.  First cloud: every Gaussian in a ball at the origin, seen
    by both views.  Second cloud: the first half stays in that ball with an opacity below 1/255 (radii > 0 in both
    views, no pairs anywhere); the second half is an opaque ball behind view 1's camera, which only view 0 sees.  So in
    the second step view 1 renders no pair, while its SplatGrad slice still holds the first step's sums unless zeroed."""
    from gs_b200 import camera, optim_step
    g = torch.Generator().manual_seed(41)
    vnp = camera.orbit_views(2, W, H)
    views = optim_step.ViewSet(vnp, W, H, DEG, dev)
    vm = vnp[1, :16].reshape(4, 4).astype(np.float64)                # row-vector world -> view transform
    centre = -vm[3, :3] @ np.linalg.inv(vm[:3, :3])                  # camera 1's position (at radius 1.75)
    far = torch.from_numpy(centre * (2.5 / 1.75)).float()            # 0.75 behind camera 1, on camera 0's axis
    base = dict(scales=torch.exp(torch.empty(N, 3).uniform_(np.log(0.01), np.log(0.04), generator=g)),
                rotations=torch.nn.functional.normalize(torch.randn(N, 4, generator=g), dim=1),
                shs=torch.rand(N, (DEG + 1) ** 2, 3, generator=g) - 0.5)
    first = dict(base, means3D=_ball(g, N, 0.5), opacities=torch.empty(N, 1).uniform_(0.2, 0.8, generator=g))
    second = dict(base, means3D=first["means3D"].clone(), opacities=first["opacities"].clone())
    second["means3D"][N // 2:] = far + _ball(g, N - N // 2, 0.2)
    second["opacities"][:N // 2] = DEAD_OPACITY
    dl = torch.rand(2, 5, H, W, generator=g) * 2 - 1
    dl[:, 3:] *= 0.1
    to = lambda c: optim_step.PackedParams({k: v.to(dev).contiguous() for k, v in c.items()})     # noqa: E731
    return views, to(first), to(second), dl.to(dev)


def second_step_grads(views, second, dl):
    from gs_b200 import optim_step
    optim_step.step_device_pipelined(second, views, dl)
    torch.cuda.synchronize()
    return second.grads.cpu()


def _within_one_ulp(a, b):
    m = torch.maximum(a.abs(), b.abs())
    ulp = torch.nextafter(m, torch.full_like(m, float("inf"))) - m
    return (a == b) | ((a - b).abs() <= ulp)


def test_view_without_pairs_reads_a_zeroed_slice(tmp_path):
    from gs_b200 import optim_step
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    dev = torch.device("cuda:0")
    views, first, second, dl = make_case(dev)
    radii = torch.empty(2, N, dtype=torch.int32, device=dev)
    _, pairs = optim_step.render_views(second, views, radii=radii)
    assert pairs > 0 and bool((radii[1, :N // 2] > 0).any()), "view 1 must see the dead half"
    assert not bool((radii[1, N // 2:] > 0).any()), "view 1 must not see the opaque half"
    v1 = optim_step.ViewSet(np.ascontiguousarray(views.host[1:2]), W, H, DEG, dev)
    assert optim_step.render_views(second, v1)[1] == 0, "view 1 must render no pair"

    assert optim_step.step_device_pipelined(first, views, dl) > 0       # leaves non-zero sums in both slices
    torch.cuda.synchronize()
    got = second_step_grads(views, second, dl)

    out = tmp_path / "fresh.npy"
    env = dict(os.environ, PYTHONNOUSERSITE="1")
    subprocess.run([sys.executable, os.path.abspath(__file__), str(out)], check=True, env=env, timeout=600)
    fresh = torch.from_numpy(np.load(out))
    ok = _within_one_ulp(got, fresh)
    assert bool(ok.all()), f"{int((~ok).sum())} of {ok.numel()} gradient elements differ from a fresh process"
    # the dead half has zero sums in every view, so all its gradients are zero
    o, dead = 0, N // 2
    for w in (3, 3 * (DEG + 1) ** 2, 1, 3, 4, 3):
        rows = got[o:o + w * N].view(N, w)
        assert bool((rows[:dead] == 0).all()), "a Gaussian without pairs received gradient"
        assert bool((rows[dead:] != 0).any())
        o += w * N


if __name__ == "__main__":          # the fresh process: the second step only
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(root, "comfyui-3d-pack_b200"), root]
    views_, _, second_, dl_ = make_case(torch.device("cuda:0"))
    np.save(sys.argv[1], second_step_grads(views_, second_, dl_).numpy())
