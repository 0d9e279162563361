"""Hunyuan3D's custom_rasterizer drop-in on the GPU: bit-exact against the reference's own outputs (the golden fixture,
and the reference's CUDA binaries in oracle/_ref at the pipelines' sizes), the faces the reference is undefined on,
and interpolate's values, gradients and run-to-run bits."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import build_ref
from oracle import cr_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RASTER, INTERP = O.golden_cases(os.path.join(ROOT, "tests", "golden", "ref_custom_rasterizer.npz"))
DEV = torch.device("cuda:0")


def _cr():
    import custom_rasterizer
    return custom_rasterizer


def _raster(pos, tri, hw, depth=None):
    cr = _cr()
    pos = torch.as_tensor(pos, device=DEV)[None]
    tri = torch.as_tensor(tri, device=DEV)
    if depth is None:
        return cr.rasterize(pos, tri, hw)
    return cr.rasterize(pos, tri, hw, torch.as_tensor(depth, device=DEV), 1)


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32).cpu(), b.contiguous().view(torch.int32).cpu())


@pytest.mark.parametrize("name", sorted(RASTER))
def test_golden_rasterize_bit_exact(name):
    c = RASTER[name]
    fi, b = _raster(c["pos"], c["tri"], c["hw"], c["depth"])
    fi, b = fi.cpu().numpy(), b.cpu().numpy()
    if c["digest"] is not None:
        assert O.digest(fi, b) == c["digest"]
    else:
        assert np.array_equal(fi, c["findices"])
        assert np.array_equal(b.view(np.uint32), c["bary"].view(np.uint32))


@pytest.mark.parametrize("name", sorted(INTERP))
def test_golden_interpolate_bit_exact(name):
    """MeshRender's sequence: rasterize -> cat into a float rast_out -> slice -> interpolate (or int32 ids)."""
    c = INTERP[name]
    r = RASTER[c["src"]]
    fi, b = _raster(r["pos"], r["tri"], r["hw"], r["depth"])
    tri = torch.as_tensor(r["tri"], device=DEV)
    tri = tri.long() if c["tri_i64"] else tri
    col = torch.as_tensor(c["col"], device=DEV)
    if c["fp32_ids"]:
        rast_out = torch.cat((b, fi.unsqueeze(-1)), dim=-1).unsqueeze(0)
        out = _cr().interpolate(col, rast_out[0, ..., -1], rast_out[0, ..., :-1], tri)
    else:
        out = _cr().interpolate(col, fi, b, tri)
    out = out.cpu().numpy()
    if c["out_digest"] is not None:
        assert hashlib.sha256(out.tobytes()).hexdigest() == c["out_digest"]
    else:
        assert np.array_equal(out.view(np.uint32), c["out"].view(np.uint32))


def test_undefined_faces_are_skipped():
    """A face with a NaN, infinite or out-of-int-range vertex, or a bad vertex id, leaves every pixel as without it."""
    c = RASTER["mixed_40x31"]
    pos = np.concatenate([c["pos"], np.array([[np.nan, 0.1, 0.2, 1.0], [0.2, np.inf, 0.2, 1.0], [3e9, 0.3, 0.1, 1.0],
                                              [0.1, -2e12, 0.1, 1.0]], np.float32)])
    N = c["pos"].shape[0]
    extra = np.array([[N, 0, 1], [2, N + 1, 3], [N + 2, 4, 5], [6, 7, N + 3], [0, 1, 10 ** 6], [-1, 2, 3]], np.int32)
    base = _raster(c["pos"], c["tri"], c["hw"])
    fi, b = _raster(pos, np.concatenate([c["tri"], extra]), c["hw"])
    assert torch.equal(fi, base[0]) and _bits_equal(b, base[1])
    assert np.array_equal(fi.cpu().numpy(), c["findices"])


# ---- against the numpy oracle, through every queue of cr_large_kernel ------------------------------------------------
# cr_raster.cu: boxes above 256 pixels go to the warp queue, above CTA_AREA to the CTA queue; the CTA queue splits each
# face over gridDim.x / n CTAs when it holds n <= GRID faces, and hands out whole faces otherwise.
CTA_AREA, GRID = 8192, 132 * 8


def large_faces(n, hw, seed):
    """n random faces spanning most of an hw image, a few vertices with w < 0 and some with negative depth."""
    g = torch.Generator().manual_seed(seed)
    N = n + 16
    pos = torch.cat([torch.rand(N, 3, generator=g) * 2.6 - 1.3, torch.rand(N, 1, generator=g) * 1.2 + 0.4], 1)
    pos[:8, 3] *= -1
    pos[8:16, 2] = -2.5 * pos[8:16, 3]
    tri = torch.randint(0, N, (n, 3), generator=g, dtype=torch.int32)
    return pos, tri, hw


def oracle_cases():
    xyz, tri, uv = sphere(20000, seed=4)
    sf_pos, sf_tri = screen_filling()
    return {"screen_filling_256": (sf_pos, sf_tri, (256, 256), None),
            "screen_filling_211x300_prior": (sf_pos, sf_tri, (211, 300), 5),
            "view384_20k": (view_pos(xyz, (384, 384)), tri, (384, 384), None),
            "uv512_20k_prior": (uv_pos(uv), tri, (512, 512), 6),
            "large_300_256x192": large_faces(300, (192, 256), 7) + (None,),
            "large_1000_256x192_prior": large_faces(1000, (192, 256), 8) + (9,),
            "large_1800_256x192": large_faces(1800, (192, 256), 10) + (None,)}


def _cta_queue_length(pos, tri, hw):
    valid, xlo, xhi, ylo, yhi = O.face_boxes(pos.numpy(), tri.numpy(), hw[1], hw[0])
    area = np.clip(xhi - xlo + 1, 0, None) * np.clip(yhi - ylo + 1, 0, None)
    return int((valid & (area > CTA_AREA)).sum())


def test_oracle_cases_reach_every_cta_queue_mode():
    n = {k: _cta_queue_length(*c[:3]) for k, c in oracle_cases().items()}
    assert 0 < n["screen_filling_256"] <= GRID // 2                 # split, several CTAs per face
    assert 0 < n["large_300_256x192"] <= GRID // 2
    assert GRID // 2 < n["large_1000_256x192_prior"] <= GRID        # split, one CTA per face, spare CTAs idle
    assert n["large_1800_256x192"] > GRID                          # whole faces, CTAs take turns
    assert n["view384_20k"] == 0


ORACLE_CASES = ["screen_filling_256", "screen_filling_211x300_prior", "view384_20k", "uv512_20k_prior",
                "large_300_256x192", "large_1000_256x192_prior", "large_1800_256x192"]


@pytest.mark.parametrize("case", ORACLE_CASES)
def test_oracle_bit_exact(case):
    pos, tri, hw, prior = oracle_cases()[case]
    depth = None if prior is None else _prior(hw, prior)
    fi, b = _raster(pos, tri, hw, depth)
    ofi, ob = O.rasterize(pos.numpy(), tri.numpy(), hw[1], hw[0], None if depth is None else depth.cpu().numpy())
    assert int((ofi != 0).sum()) > 0
    fi, b = fi.cpu().numpy(), b.cpu().numpy()
    assert np.array_equal(fi, ofi), f"{int((fi != ofi).sum())} findices differ"
    assert np.array_equal(b.view(np.uint32), ob.view(np.uint32))


# ---- against the reference's CUDA binaries --------------------------------------------------------------------------
def _ref(variant):
    mod = build_ref.load(variant)
    if mod is None:
        pytest.skip(f"oracle/_ref has no {variant} reference build (no ComfyUI-3D-Pack checkout was found: see oracle/build_ref.py)")
    return mod


def sphere(n_faces, seed=0, noise=0.1):
    """A seeded bumpy UV sphere with about n_faces faces: (vertices [N,3] fp32, faces [F,3] int32, uv [N,2] fp32).
    The radial noise is independent per vertex, so with noise=0.1 the faces are slivers whose boxes are far larger than
    a decimated scan's (4.7k pixels on average for 40k faces in a 2048^2 view); noise=0 gives a smooth sphere."""
    nu = max(4, int(round((n_faces / 2) ** 0.5)))
    nv = max(4, int(round(n_faces / (2 * (nu - 1)))) + 1)
    g = torch.Generator().manual_seed(seed)
    th = torch.linspace(0.05, np.pi - 0.05, nu, dtype=torch.float64)[:, None]
    ph = torch.linspace(0, 2 * np.pi, nv, dtype=torch.float64)[None, :]
    r = 0.45 * (1 + noise * torch.randn(nu, nv, generator=g, dtype=torch.float64).clamp(-2, 2))
    xyz = torch.stack([r * th.sin() * ph.cos(), r * th.cos().expand(nu, nv), r * th.sin() * ph.sin()], -1).reshape(-1, 3)
    i, j = torch.meshgrid(torch.arange(nu - 1), torch.arange(nv - 1), indexing="ij")
    a = (i * nv + j).reshape(-1)
    tri = torch.cat([torch.stack([a, a + nv, a + 1], 1), torch.stack([a + 1, a + nv, a + nv + 1], 1)]).int()
    uv = torch.stack([(ph / (2 * np.pi)).expand(nu, nv), (th / np.pi).expand(nu, nv)], -1).reshape(-1, 2)
    return xyz.float(), tri, uv.float()


def view_pos(xyz, hw, elev=15.0, azim=30.0, dist=1.45):
    """Perspective clip positions (49.13 degrees, near 0.01, far 100), as MeshRender's default camera."""
    f = 1.0 / np.tan(np.radians(49.13) / 2)
    n, fa = 0.01, 100.0
    proj = np.array([[f / (hw[1] / hw[0]), 0, 0, 0], [0, f, 0, 0], [0, 0, -(fa + n) / (fa - n), -2 * fa * n / (fa - n)],
                     [0, 0, -1, 0]])
    e, a = np.radians(elev), np.radians(azim)
    ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    rx = np.array([[1, 0, 0], [0, np.cos(e), -np.sin(e)], [0, np.sin(e), np.cos(e)]])
    mv = np.eye(4)
    mv[:3, :3] = rx @ ry
    mv[2, 3] = -dist
    v = np.concatenate([xyz.double().numpy(), np.ones((xyz.shape[0], 1))], 1)
    return torch.from_numpy((v @ (proj @ mv).T).astype(np.float32))


def uv_pos(uv):
    return torch.cat([uv * 2 - 1, torch.zeros(uv.shape[0], 1), torch.ones(uv.shape[0], 1)], 1)


def screen_filling():
    """A few triangles that each cover most of a 2048^2 view, at distinct and equal depths."""
    pos = torch.tensor([[-1.5, -1.5, 0.2, 1], [3.0, -1.2, 0.3, 1], [-1.1, 3.0, 0.1, 1], [1.4, 1.3, -0.1, 1],
                        [-1.3, 1.2, 0.25, 1], [1.2, -1.4, 0.25, 1], [0.9, 0.95, 0.4, 1.2], [-0.8, -0.9, 0.3, 0.9]])
    tri = torch.tensor([[0, 1, 2], [3, 4, 5], [0, 5, 6], [4, 7, 1], [2, 3, 7], [0, 1, 2]], dtype=torch.int32)
    return pos, tri


def pipeline_cases():
    xyz40, tri40, uv40 = sphere(40000, seed=1)
    xyz500, tri500, _ = sphere(500000, seed=2)
    sf_pos, sf_tri = screen_filling()
    return {"view2048_40k": (view_pos(xyz40, (2048, 2048)), tri40, (2048, 2048)),
            "view2048_500k": (view_pos(xyz500, (2048, 2048)), tri500, (2048, 2048)),
            "uv4096_40k": (uv_pos(uv40), tri40, (4096, 4096)),
            "screen_filling_2048": (sf_pos, sf_tri, (2048, 2048))}


CASES = ["view2048_40k", "view2048_500k", "uv4096_40k", "screen_filling_2048"]


@pytest.fixture(scope="module")
def pipelines():
    return pipeline_cases()


def _prior(hw, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(hw, generator=g) * 2 - 1).to(DEV)      # skips about half of the covered pixels


def _ref_run(mod, pos, tri, hw, depth):
    D = depth if depth is not None else torch.zeros(0, device=DEV)
    fi, b = mod.rasterize_image(pos.to(DEV), tri.to(DEV), D, hw[1], hw[0], 1e-6, int(depth is not None))
    torch.cuda.synchronize()
    return fi, b


@pytest.mark.parametrize("prior", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_reference_nofma_cuda_bit_exact(pipelines, case, prior):
    ref = _ref("nofma")
    pos, tri, hw = pipelines[case]
    depth = _prior(hw, 3) if prior else None
    rfi, rb = _ref_run(ref, pos, tri, hw, depth)
    fi, b = _raster(pos, tri, hw, depth)
    assert int((fi != 0).sum()) > 0
    assert torch.equal(fi, rfi), f"{int((fi != rfi).sum())} findices differ"
    assert _bits_equal(b, rb)


@pytest.mark.parametrize("case", CASES)
def test_reference_default_cuda_disagrees_only_where_its_builds_do(pipelines, case):
    """The default (FMA-contracted) reference build differs from ours only on pixels where it also differs from the
    reference's own nofma build."""
    ref_d, ref_n = _ref("default"), _ref("nofma")
    pos, tri, hw = pipelines[case]
    dfi, _ = _ref_run(ref_d, pos, tri, hw, None)
    nfi, _ = _ref_run(ref_n, pos, tri, hw, None)
    fi, _ = _raster(pos, tri, hw)
    ours, builds = fi != dfi, nfi != dfi
    print(f"{case}: findices differ from the default build on {int(ours.sum())} pixels; "
          f"the two reference builds differ on {int(builds.sum())}")
    assert not bool((ours & ~builds).any())


# ---- interpolate --------------------------------------------------------------------------------------------------
def _interp_inputs(seed=0, hw=(256, 192), C=3, fp32_ids=True):
    xyz, tri, _ = sphere(20000, seed=seed)
    fi, b = _raster(view_pos(xyz, hw), tri, hw)
    g = torch.Generator().manual_seed(seed)
    col = torch.randn(1, xyz.shape[0], C, generator=g).to(DEV)
    ids = fi.float() if fp32_ids else fi
    return col, ids, b, tri.to(DEV)


def _torch_expr(col, findices, barycentric, tri):
    f = findices - 1 + (findices == 0)
    vcol = col[0, tri.long()[f.long()]]
    return torch.sum(barycentric.view(*barycentric.shape, 1) * vcol, axis=-2).view(1, *barycentric.shape[:2], -1)


@pytest.mark.parametrize("fp32_ids", [False, True])
@pytest.mark.parametrize("C", [1, 3, 4])
def test_interpolate_matches_torch_expression(C, fp32_ids):
    col, ids, b, tri = _interp_inputs(C=C, fp32_ids=fp32_ids)
    out = _cr().interpolate(col, ids, b, tri)
    ref = _torch_expr(col, ids, b, tri)
    assert out.shape == ref.shape
    # torch on the GPU may add the three corners in another order: two orders of a 3-term fp32 sum differ by at most
    # 4u sum|t| (u = 2^-24), one ulp of the largest |term| scale, however much the terms cancel
    f = (ids - 1 + (ids == 0)).long()
    mag = torch.sum(b.abs()[..., None] * col[0, tri.long()[f]].abs(), -2)[None]
    assert bool((torch.abs(out - ref) <= mag * 2.0 ** -22).all())
    assert torch.equal(out, _torch_expr(col.cpu(), ids.cpu(), b.cpu(), tri.cpu()).to(DEV))


def test_interpolate_gradients():
    col, ids, b, tri = _interp_inputs(C=3)
    col.requires_grad_(True)
    bq = b.clone().requires_grad_(True)
    g = torch.randn(1, *b.shape[:2], 3, generator=torch.Generator().manual_seed(5)).to(DEV)
    runs = []
    for _ in range(2):
        col.grad = bq.grad = None
        (_cr().interpolate(col, ids, bq, tri) * g).sum().backward()
        runs.append((col.grad.clone(), bq.grad.clone()))
    assert _bits_equal(runs[0][0], runs[1][0]) and _bits_equal(runs[0][1], runs[1][1])
    # col: float64 scatter of b_k * g onto the face's vertices
    f = (ids - 1 + (ids == 0)).long()
    v = tri.long()[f].reshape(-1)
    contrib = (b.double()[..., :, None] * g[0].double()[..., None, :]).reshape(-1, 3)
    ref = torch.zeros(col.shape[1], 3, dtype=torch.float64, device=DEV).index_add_(0, v, contrib)
    rel = float((runs[0][0][0].double() - ref).norm() / ref.norm())
    assert rel < 1e-6, rel
    # barycentric: the torch expression's own gradient
    b2 = b.clone().requires_grad_(True)
    (_torch_expr(col.detach(), ids, b2, tri) * g).sum().backward()
    assert torch.allclose(runs[0][1], b2.grad, rtol=1e-6, atol=1e-6)


def test_refusals_on_gpu():
    cr = _cr()
    pos = torch.zeros(1, 3, 4, device=DEV)
    with pytest.raises(TypeError):
        cr.rasterize(pos, torch.zeros(1, 3, dtype=torch.int64, device=DEV), (8, 8))
    with pytest.raises(TypeError):
        cr.rasterize(pos.double(), torch.zeros(1, 3, dtype=torch.int32, device=DEV), (8, 8))
    with pytest.raises(ValueError):
        cr.rasterize(pos, torch.zeros(1, 3, dtype=torch.int32, device=DEV), (8, 8), torch.zeros(0, device=DEV), 1)


def test_no_faces_and_side_stream():
    cr = _cr()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fi, b = cr.rasterize(torch.zeros(1, 3, 4, device=DEV), torch.zeros(0, 3, dtype=torch.int32, device=DEV), (5, 7))
    s.synchronize()
    assert fi.shape == (5, 7) and b.shape == (5, 7, 3)
    assert not bool(fi.any()) and not bool(b.any())
