"""GPU tests of the point rasterizer and points_projection (gs_b200.points, csrc/pts_raster.cu) against the brute-force
numpy oracle (oracle/points_oracle.py).  Fragments are compared element for element, bit for bit."""
import numpy as np
import pytest
import torch

from oracle import points_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
f32 = np.float32


def _P():
    from gs_b200 import points
    return points


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _eq(got, want, what=""):
    g = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    w = np.asarray(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    if g.dtype == np.float32:
        g, w = g.view(np.uint32), w.astype(f32).view(np.uint32)
    bad = np.argwhere(g != w)
    assert bad.size == 0, f"{what}: {len(bad)} differ, first at {bad[:3].tolist()}"


def _look_at(rng, n, dist=2.0):
    """n OpenCV camera-to-world matrices on a sphere of radius `dist`, looking at the origin (TGS's setup)."""
    out = []
    for _ in range(n):
        eye = rng.normal(size=3)
        eye *= dist / np.linalg.norm(eye)
        fwd = -eye / np.linalg.norm(eye)
        right = np.cross(fwd, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        c2w = np.eye(4)
        c2w[:3, :3] = np.stack([right, down, fwd], 1)
        c2w[:3, 3] = eye
        out.append(c2w)
    return np.array(out, f32)


def _intrinsics(n, H, W, fov=40.0):
    f = 0.5 * H / np.tan(np.radians(fov) / 2)
    return np.repeat(np.array([[[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]]], f32), n, 0)


def _cameras(rng, n, H, W):
    """(R, T, Km) fp32 numpy world-to-camera cameras, and the matching gs_b200 cameras."""
    w2c = np.linalg.inv(_look_at(rng, n).astype(np.float64)).astype(f32)
    R, T, Km = np.ascontiguousarray(w2c[:, :3, :3]), np.ascontiguousarray(w2c[:, :3, 3]), _intrinsics(n, H, W)
    size = torch.tensor([[H, W]] * n, device=DEV)
    return (R, T, Km), _P().cameras_from_opencv_projection(_t(R), _t(T), _t(Km), size)


def _run(clouds, cams, H, W, radius, K, padded=False):
    P = _P()
    pc = P.Pointclouds(_t(np.stack(clouds)) if padded else [_t(c) for c in clouds])
    s = P.PointsRasterizationSettings(image_size=(H, W), radius=radius, points_per_pixel=K, bin_size=0)
    return P.PointsRasterizer(cameras=cams, raster_settings=s)(pc)


def _check(clouds, np_cams, cams, H, W, radius, K, padded=False):
    fr = _run(clouds, cams, H, W, radius, K, padded)
    want = O.rasterize(clouds, *np_cams, None, H, W, radius, K)
    for got, w, nm in zip(fr, want, ("idx", "zbuf", "dists")):
        _eq(got, w, nm)
    return fr, want


def _cloud(rng, n, span=0.5):
    return ((rng.random((n, 3)) * 2 - 1) * span).astype(f32)


@pytest.mark.parametrize("Np", [2048, 16384])
def test_tgs_sizes_match_the_oracle(Np):
    rng = np.random.default_rng(Np)
    np_cams, cams = _cameras(rng, 1, 252, 252)
    fr, want = _check([_cloud(rng, Np)], np_cams, cams, 252, 252, 0.0075, 1, padded=True)
    assert (want[0] >= 0).sum() > 1000
    assert fr.idx.dtype == torch.int32 and fr.idx.shape == (1, 252, 252, 1)


@pytest.mark.parametrize("K", [1, 2, 8])
def test_k_nearest_match_the_oracle(K):
    rng = np.random.default_rng(K)
    np_cams, cams = _cameras(rng, 1, 64, 80)
    fr, want = _check([_cloud(rng, 3000)], np_cams, cams, 64, 80, 0.05, K)
    assert (want[0][..., K - 1] >= 0).sum() > 100


def _simple(n, H, W):
    """R = I, T = 0, fx = fy = s, principal point at the centre: the world point (-a z, -b z, z) lands at NDC (a, b)."""
    s = min(H, W) / 2
    Km = np.repeat(np.array([[[s, 0, W / 2], [0, s, H / 2], [0, 0, 1]]], f32), n, 0)
    R, T = np.repeat(np.eye(3, dtype=f32)[None], n, 0), np.zeros((n, 3), f32)
    return (R, T, Km), _P().cameras_from_opencv_projection(_t(R), _t(T), _t(Km), torch.tensor([[H, W]] * n, device=DEV))


def _world(a, b, z):
    return np.stack([-a * z, -b * z, z], -1).astype(f32)


@pytest.mark.parametrize("K", [1, 2])
def test_points_straddling_pixel_centre_boundaries(K):
    """Points on the midlines between pixel centres and at exactly +-radius from centres, along both axes."""
    H, W = 48, 64
    xc, yc = O.centres(H, W)
    xm, ym = (xc[:-1] + xc[1:]) / 2, (yc[:-1] + yc[1:]) / 2
    r = f32(2.0 / H * 0.75)
    rng = np.random.default_rng(7)
    a = np.concatenate([xm, xc + r, xc - r, xm[: H - 1]]).astype(f32)
    b = np.concatenate([rng.choice(yc, len(xm)), rng.choice(yc, 2 * W), ym]).astype(f32)
    z = rng.choice(f32([1.0, 1.5, 2.0]), len(a))
    np_cams, cams = _simple(1, H, W)
    fr, want = _check([_world(a, b, z)], np_cams, cams, H, W, float(r), K)
    assert (want[0] >= 0).sum() > 200


@pytest.mark.parametrize("K", [1, 2, 8])
def test_all_points_on_one_pixel(K):
    rng = np.random.default_rng(3)
    n = 4000
    z = rng.choice(f32([1.0, 1.25, 1.5, 2.0]), n)                   # many exact z ties
    pts = _world(np.full(n, 0.01, f32), np.full(n, -0.02, f32), z)
    np_cams, cams = _simple(1, 32, 32)
    fr, want = _check([pts], np_cams, cams, 32, 32, 0.03, K)
    assert (want[0][..., 0] >= 0).sum() >= 1


def test_ragged_clouds_with_empty_ones_and_shared_camera():
    rng = np.random.default_rng(11)
    H, W = 40, 56
    clouds = [_cloud(rng, 700), np.zeros((0, 3), f32), _cloud(rng, 1), _cloud(rng, 1500)]
    np_cams, cams = _cameras(rng, 4, H, W)
    _check(clouds, np_cams, cams, H, W, 0.04, 2)
    np1, cam1 = _cameras(rng, 1, H, W)                             # one camera for every cloud
    _check(clouds, np1, cam1, H, W, 0.04, 3)
    _check([_cloud(rng, 500), _cloud(rng, 500)], np1, cam1, H, W, 0.04, 1, padded=True)


def test_empty_clouds():
    P = _P()
    np_cams, cams = _simple(2, 16, 24)
    fr = _run([np.zeros((0, 3), f32)] * 2, cams, 16, 24, 0.1, 2, padded=True)
    assert fr.idx.shape == (2, 16, 24, 2) and (fr.idx == -1).all() and (fr.zbuf == -1).all() and (fr.dists == -1).all()
    fr = _run([np.zeros((0, 3), f32)] * 2, cams, 16, 24, 0.1, 1)
    assert (fr.idx == -1).all()
    _, cam1 = _simple(1, 8, 8)
    fr = P.PointsRasterizer(cam1, P.PointsRasterizationSettings(8, 0.1, 1))(P.Pointclouds(torch.zeros(0, 5, 3, device=DEV)))
    assert fr.idx.shape == (0, 8, 8, 1)


def _tgs_inputs(rng, B, Np, C, H=252, W=252):
    pts = _t(_cloud(rng, B * Np).reshape(B, Np, 3))
    c2w = _t(_look_at(rng, B))
    K = _t(_intrinsics(B, H, W))
    feat = _t(rng.normal(size=(B, C, H, W)).astype(f32))
    return pts, c2w, K, feat


def _oracle_idx(pts, c2w, K, H, W, radius, k):
    """idx from the oracle, with the camera the fused path uses (the device inverse, rounded to fp32)."""
    w2c = torch.linalg.inv_ex(c2w)[0].cpu().numpy()
    R, T = np.ascontiguousarray(w2c[:, :3, :3]), np.ascontiguousarray(w2c[:, :3, 3])
    return O.rasterize(list(pts.cpu().numpy()), R, T, K.cpu().numpy(), None, H, W, radius, k)[0]


@pytest.mark.parametrize("B,Np,K", [(1, 16384, 1), (2, 2048, 2)])
def test_points_projection_lift_matches_the_oracle_and_repeats(B, Np, K):
    P = _P()
    rng = np.random.default_rng(B * Np + K)
    pts, c2w, Km, feat = _tgs_inputs(rng, B, Np, 24)
    out = P.points_projection(pts, c2w, Km, feat, 0.0075, K)
    assert out.shape == (B, Np, 24) and out.dtype == torch.float32
    idx = _oracle_idx(pts, c2w, Km, 252, 252, 0.0075, K)
    want = O.lift(idx, feat.cpu().numpy(), B * Np).reshape(B, Np, 24)
    _eq(out, want, "lift")
    multi = np.bincount(idx[idx >= 0], minlength=B * Np)
    assert (multi > 1).sum() > 100                                 # the largest-pixel rule decides for these
    for _ in range(10):
        _eq(P.points_projection(pts, c2w, Km, feat, 0.0075, K), out.cpu().numpy(), "rerun")


def test_lift_reads_strided_and_half_features():
    P = _P()
    rng = np.random.default_rng(5)
    pts, c2w, Km, feat = _tgs_inputs(rng, 1, 4096, 16, 96, 128)
    base = P.points_projection(pts, c2w, Km, feat, 0.02)
    nhwc = feat.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)   # same values, channels-last strides
    _eq(P.points_projection(pts, c2w, Km, nhwc, 0.02), base.cpu().numpy(), "strided")
    half = feat.half()
    _eq(P.points_projection(pts, c2w, Km, half, 0.02), P.points_projection(pts, c2w, Km, half.float(), 0.02).cpu().numpy(),
        "half")


def _lift64(idx, P, K):
    """The oracle's lift as a float64 torch function of the features, for autograd and finite differences."""
    N, H, W, _ = idx.shape
    win = torch.from_numpy(O.winners(idx, P))
    sel = win >= 0
    pix = win[sel] // K

    def f(x):
        out = torch.zeros(P, x.size(1), dtype=torch.float64)
        out[sel] = x.permute(0, 2, 3, 1).reshape(N * H * W, -1)[pix]
        return out
    return f


@pytest.mark.parametrize("K", [1, 2])
def test_lift_backward(K):
    P = _P()
    rng = np.random.default_rng(20 + K)
    B, Np, C, H, W = 2, 3000, 5, 48, 64
    pts, c2w, Km, feat = _tgs_inputs(rng, B, Np, C, H, W)
    radius = 0.06
    f = feat.clone().requires_grad_(True)
    out = P.points_projection(pts, c2w, Km, f, radius, K)
    g = _t(rng.normal(size=out.shape).astype(f32))
    out.backward(g)
    grad = f.grad.clone()
    idx = _oracle_idx(pts, c2w, Km, H, W, radius, K)
    g64 = g.cpu().double().reshape(B * Np, C)
    want = O.lift_backward(idx, g64.numpy(), C, B * Np)
    x64 = feat.cpu().double().requires_grad_(True)
    (auto,) = torch.autograd.grad(_lift64(idx, B * Np, K)(x64), x64, g64)
    np.testing.assert_array_equal(auto.numpy(), want)
    if K == 1:
        _eq(grad, want, "grad")                                      # one term per pixel: exact
    else:
        np.testing.assert_allclose(grad.cpu().numpy(), want, rtol=1e-6, atol=1e-6)
    for _ in range(3):
        f.grad = None
        P.points_projection(pts, c2w, Km, f, radius, K).backward(g)
        _eq(f.grad, grad.cpu().numpy(), "rerun grad")


@pytest.mark.parametrize("K", [1, 2])
def test_lift_backward_against_finite_differences(K):
    """gradcheck in float64: the kernel's backward, moved to float64, against central differences of the oracle's lift
    on the kernel's own fragments."""
    P = _P()
    rng = np.random.default_rng(40 + K)
    B, Np, C, H, W = 1, 400, 2, 10, 14
    pts, c2w, Km, feat = _tgs_inputs(rng, B, Np, C, H, W)
    f = feat.clone().requires_grad_(True)
    out = P.points_projection(pts, c2w, Km, f, 0.12, K)
    idx = _oracle_idx(pts, c2w, Km, H, W, 0.12, K)
    assert (idx >= 0).sum() > 50
    lift = _lift64(idx, B * Np, K)

    class Kernel(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x):
            return lift(x)

        @staticmethod
        def backward(ctx, go):
            (gx,) = torch.autograd.grad(out, f, go.reshape(out.shape).to(DEV, torch.float32), retain_graph=True)
            return gx.cpu().double()

    x = feat.cpu().double().requires_grad_(True)
    assert torch.autograd.gradcheck(Kernel.apply, (x,), eps=1e-3, atol=1e-5, rtol=1e-4)


def test_replaying_tgs_points_projection_with_the_substituted_imports():
    """TriplaneGaussian's utils/ops.py points_projection, restated step by step on the names gs_b200.points provides
    (its import block substituted), gives the fused function's output.  Its index_put leaves an undefined winner on
    CUDA where a point covers several pixels, so the replay's lift is done sequentially on the CPU, which is the
    largest-pixel rule; the CUDA index_put result is checked where it is defined."""
    from gs_b200.points import (PointsRasterizationSettings, PointsRasterizer, Pointclouds,
                                cameras_from_opencv_projection, points_projection)
    rng = np.random.default_rng(9)
    points, c2ws, intrinsics, local_features = _tgs_inputs(rng, 1, 16384, 32)
    B, C, H, W = local_features.shape
    Np = points.shape[1]
    settings = PointsRasterizationSettings(image_size=(H, W), radius=0.0075, points_per_pixel=1, bin_size=0)
    w2cs = torch.inverse(c2ws)
    image_size = torch.as_tensor([H, W]).view(1, 2).expand(w2cs.shape[0], -1).to(DEV)
    cameras = cameras_from_opencv_projection(w2cs[:, :3, :3], w2cs[:, :3, 3], intrinsics, image_size)
    fragments = PointsRasterizer(cameras=cameras, raster_settings=settings)(Pointclouds(points))
    idx = fragments.idx.long()
    visible = idx > -1
    target = idx[visible]
    values = local_features.permute(0, 2, 3, 1).unsqueeze(-2).expand(-1, -1, -1, 1, -1)[visible]
    seq = torch.zeros(B * Np, C)
    for t, v in zip(target.cpu().tolist(), values.cpu()):
        seq[t] = v                                                  # index_put in order: the last write stays
    fused = points_projection(points, c2ws, intrinsics, local_features)
    _eq(fused.reshape(B * Np, C), seq.numpy(), "replay")
    proj = torch.zeros(B * Np, C, device=DEV)
    proj[target] = values
    once = torch.bincount(target, minlength=B * Np) == 1
    assert int(once.sum()) > 1000
    _eq(fused.reshape(B * Np, C)[once], proj[once].cpu().numpy(), "index_put where defined")


def test_errors_inference_mode_and_side_stream():
    P = _P()
    rng = np.random.default_rng(2)
    pts, c2w, Km, feat = _tgs_inputs(rng, 2, 512, 4, 32, 40)
    with pytest.raises(ValueError):
        P.points_projection(pts, c2w, Km, feat[:1])
    with pytest.raises(ValueError):
        P.points_projection(pts, c2w[:, :3], Km, feat)
    with pytest.raises(ValueError):
        P.points_projection(pts, c2w, Km[:, :2], feat)
    with pytest.raises(ValueError):
        P.points_projection(pts[..., :2], c2w, Km, feat)
    with pytest.raises(NotImplementedError):
        P.points_projection(pts, c2w, Km, feat, 0.01, 9)
    with pytest.raises(TypeError):
        P.points_projection(pts.double(), c2w, Km, feat)
    with pytest.raises(RuntimeError, match="CPU"):
        P.points_projection(pts, c2w, Km, feat.cpu())
    with pytest.raises(ValueError):
        P.Pointclouds([pts[0, :, :2]])
    with pytest.raises(ValueError):
        P.cameras_from_opencv_projection(c2w[:, :3, :3], c2w[:1, :3, 3], Km, torch.ones(2, 2, device=DEV))
    _, cams3 = _cameras(rng, 3, 32, 40)
    with pytest.raises(ValueError, match="cameras"):
        P.PointsRasterizer(cams3, P.PointsRasterizationSettings((32, 40), 0.1, 1))(P.Pointclouds(pts))

    base = P.points_projection(pts, c2w, Km, feat, 0.03, 2)
    with torch.inference_mode():
        _eq(P.points_projection(pts, c2w, Km, feat, 0.03, 2), base.cpu().numpy(), "inference mode")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = P.points_projection(pts, c2w, Km, feat, 0.03, 2)
    torch.cuda.current_stream().wait_stream(side)
    _eq(got, base.cpu().numpy(), "side stream")
