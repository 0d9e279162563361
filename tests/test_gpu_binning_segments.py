"""The multi-view entries bin all views of a chunk in segmented launches (one segment per view): depth sort,
gather-scan, emit, tile sort and ranges each cover every view at once.  A scene built to hit the segment edges must
render exactly what the single-view entry renders, view by view."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _depth_top_digit_trivial(vnp, means):
    """Whether the depth sort's top digit is the same for every Gaussian of the view: view-space z as fp32 bits,
    Gaussians behind the near plane keyed 0xFFFFFFFF, less the view's smallest visible key."""
    m = vnp[:16].astype(np.float32)
    tz = means[:, 0] * m[2] + means[:, 1] * m[6] + means[:, 2] * m[10] + m[14]
    keys = np.where(tz > 0.2, tz.astype(np.float32).view(np.uint32), np.uint32(0xFFFFFFFF)).astype(np.uint64)
    vis = tz > 0.2
    if not vis.any():
        return None
    top = ((keys - keys[vis].min()) >> 24) & 0xFF
    return bool((top == top[0]).all())


def test_render_views_segment_edges_match_single_view_entry(dev):
    from gs_b200 import camera, optim_step, synthetic
    from gs_b200 import rasterizer as R
    N, W, H, deg = 9001, 256, 192, 1            # N: two full depth-sort partitions of 4096 and a partial one
    cloud = synthetic.make_cloud("D1", N, deg, seed=21, device=dev)
    means = cloud["means3D"]
    cloud["means3D"] = (means * (0.45 / float(means.norm(dim=1).max()))).contiguous()    # inside a 0.45 ball
    params = optim_step.PackedParams(cloud)
    far = camera.orbit_views(4, W, H, radius=1.75)             # the whole cloud 1.3..2.2 in front: top digit trivial
    near = camera.orbit_views(1, W, H, radius=0.3, azimuth_offset=20.0)   # camera inside the cloud: many more pairs
    empty = camera.orbit_views(1, W, H, radius=1.75, azimuth_offset=45.0).copy()
    empty[0, 14] = -50.0                                       # every z_view <= 0.2: no pairs at all
    vnp = np.ascontiguousarray(np.concatenate([far[0:1], near, far[1:2], empty, far[2:4]], axis=0))
    V = vnp.shape[0]
    mh = params.means3D.cpu().numpy()
    assert _depth_top_digit_trivial(vnp[0], mh) is True
    assert _depth_top_digit_trivial(vnp[1], mh) is False
    views = optim_step.ViewSet(vnp, W, H, deg, dev)
    images = torch.empty(V, 5, H, W, device=dev)
    radii = torch.empty(V, N, dtype=torch.int32, device=dev)
    _, pairs = optim_step.render_views(params, views, images, radii)
    assert int((radii[3] > 0).sum()) == 0 and float(images[3, 4].abs().max()) == 0.0
    for v in range(V):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        rs = R.GaussianRasterizationSettings(H, W, float(vnp[v, 38]), float(vnp[v, 39]), t(vnp[v, 35:38]), 1.0,
                                            t(vnp[v, :16]).view(4, 4), t(vnp[v, 16:32]).view(4, 4), deg,
                                            t(vnp[v, 32:35]), False, False)
        with torch.no_grad():
            col, rad, dep, alp = R.GaussianRasterizer(rs)(
                means3D=params.means3D, means2D=torch.zeros(N, 3, device=dev), shs=params.shs, colors_precomp=None,
                opacities=params.opacities, scales=params.scales, rotations=params.rotations)
        assert torch.equal(rad, radii[v]), f"view {v}: radii"
        assert torch.equal(col, images[v, :3]) and torch.equal(dep, images[v, 3:4]) and torch.equal(alp, images[v, 4:5]), \
            f"view {v}: image"
    # the near view carries far more pairs than the others: compare by visible-splat footprint through the radii
    foot = [(radii[v].clamp(min=0).double() ** 2).sum().item() for v in range(V)]
    assert foot[1] > 4 * max(foot[v] for v in (0, 2, 4, 5))
    assert pairs > 0
