"""Dual marching cubes on the H100 (csrc/ngp_dmc.cu via gs_b200.isosurface.DiffDMC and the `diso` shim) against the
float64 oracle (oracle/dmc_oracle.py, run on the GPU): topology exact (vertex and quad counts, quad indices element
for element), vertices within 1e-6 x the largest dimension in index units, triangles exact on every quad whose split
margin on the returned vertices exceeds 1e-5, gradients within 1e-4 relative L2, and outputs and gradients bit-identical from run to run."""
import numpy as np
import pytest
import torch

from conftest import ROOT  # noqa: F401
from oracle import dmc_oracle as D

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
MARGIN = 1e-5


def _dmc():
    from diso import DiffDMC
    return DiffDMC(dtype=torch.float32).to(DEV)


def _scale(shape, normalize):
    return torch.tensor([d - 1 for d in shape], dtype=torch.float64, device=DEV) if normalize else 1.0


def _check(grid, deform=None, iso=0.0, return_quads=False, normalize=True):
    """GPU result against the oracle; returns (verts, faces) of the GPU."""
    v, f = _dmc()(grid, deform=deform, isovalue=iso, return_quads=return_quads, normalize=normalize)
    assert v.dtype == torch.float32 and f.dtype == torch.int32 and v.device == DEV and f.device == DEV
    ov, of, info = D.dmc(grid, deform, iso=iso, return_quads=return_quads, normalize=normalize)
    assert v.shape == ov.shape and f.shape == of.shape, (v.shape, ov.shape, f.shape, of.shape)
    if v.shape[0]:
        s = _scale(grid.shape, normalize)
        err = float(((v.double() - ov) * s).abs().max())
        assert err <= 1e-6 * max(grid.shape), err
    if return_quads:
        assert torch.equal(f.long(), of)
    else:
        # the split rule is applied to the returned fp32 vertices, so its float64 margin is taken on them: the oracle's
        # own vertices differ by fp32 rounding, which moves cosines of short edges by more than 1e-5
        g2, q = f.long().reshape(-1, 2, 3), info["quads"]
        p = v.double()[q]
        m1 = torch.maximum(D.max_cos(p[:, 0], p[:, 1], p[:, 3]), D.max_cos(p[:, 1], p[:, 2], p[:, 3]))
        m2 = torch.maximum(D.max_cos(p[:, 0], p[:, 1], p[:, 2]), D.max_cos(p[:, 0], p[:, 2], p[:, 3]))
        one = torch.stack([q[:, [0, 1, 3]], q[:, [1, 2, 3]]], 1)
        two = torch.stack([q[:, [0, 1, 2]], q[:, [0, 2, 3]]], 1)
        is_one, is_two = (g2 == one).flatten(1).all(1), (g2 == two).flatten(1).all(1)
        assert bool((is_one | is_two).all())
        sure = (m1 - m2).abs() > MARGIN
        assert torch.equal(is_one[sure], (m1 < m2)[sure])
        # and where the oracle's own margin is wide, the oracle's split
        wide = info["margin"] > 1e-2
        assert torch.equal(g2[wide], of.reshape(-1, 2, 3)[wide])
    return v, f


def test_every_case_of_a_single_cube():
    rng = np.random.default_rng(0)
    for case in range(256):
        bits = np.array([(case >> i) & 1 for i in range(8)], dtype=bool)
        vals = np.where(bits, rng.uniform(-1.0, -0.05, 8), rng.uniform(0.05, 1.0, 8)).astype(np.float32)
        g = np.empty((2, 2, 2), np.float32)
        for i in range(8):
            g[i & 1, (i >> 1) & 1, i >> 2] = vals[i]
        grid = torch.from_numpy(g).to(DEV)
        for rq in (False, True):
            _check(grid, iso=0.0, return_quads=rq)


@pytest.mark.parametrize("shape", [(17, 23, 31), (9, 40, 6)])
@pytest.mark.parametrize("with_deform", [False, True])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("return_quads", [False, True])
def test_random_grids_match_the_oracle(shape, with_deform, normalize, return_quads):
    gen = torch.Generator(device=DEV).manual_seed(sum(shape))
    grid = torch.rand(shape, generator=gen, device=DEV) * 2 - 1
    deform = (torch.rand((*shape, 3), generator=gen, device=DEV) * 2 - 1) * 0.3 if with_deform else None
    _check(grid, deform, iso=0.17, return_quads=return_quads, normalize=normalize)


def test_masked_random_grid_matches_the_oracle():
    gen = torch.Generator(device=DEV).manual_seed(5)
    grid = torch.rand((21, 19, 33), generator=gen, device=DEV) * 2 - 1
    grid[torch.rand(grid.shape, generator=gen, device=DEV) < 0.05] = float("nan")
    grid[torch.rand(grid.shape, generator=gen, device=DEV) < 0.01] = float("-inf")
    for rq in (False, True):
        _check(grid, iso=-0.1, return_quads=rq)


def test_surface_cut_by_the_border_is_closed_by_the_ring():
    n = 48
    idx = torch.stack(torch.meshgrid(*[torch.arange(n, device=DEV, dtype=torch.float32)] * 3, indexing="ij"), -1)
    grid = torch.linalg.vector_norm(idx - torch.tensor([0.4, 23.3, 47.1], device=DEV), dim=-1) - 17.5
    v, f = _check(grid, normalize=False)
    f = f.cpu().numpy()
    assert D.is_oriented_manifold(f) and D.euler_characteristic(v.shape[0], f) == 2


def test_nan_band_at_257():
    grid = D.triposg_field(257, seed=1, device=DEV, nan_band=True)
    assert torch.isnan(grid).any()
    for rq in (False, True):
        v, f = _check(grid, return_quads=rq, normalize=not rq)
        assert not torch.isnan(v).any() and int(f.min()) >= 0 and int(f.max()) < v.shape[0]


def _loss_grads(grid, deform, w_seed, normalize, return_quads=False):
    g = grid.clone().requires_grad_(True)
    d = deform.clone().requires_grad_(True)
    v, f = _dmc()(g, deform=d, isovalue=0.05, return_quads=return_quads, normalize=normalize)
    w = torch.randn(v.shape, generator=torch.Generator(device=DEV).manual_seed(w_seed), device=DEV)
    (v * w + torch.sin(3 * v)).sum().backward()
    return v.detach(), f, g.grad, d.grad, w


@pytest.mark.parametrize("normalize", [False, True])
def test_gradients_match_the_oracle_and_repeat_bit_for_bit(normalize):
    shape = (14, 18, 23)
    gen = torch.Generator(device=DEV).manual_seed(11)
    grid = torch.rand(shape, generator=gen, device=DEV) * 2 - 1
    grid[3, 4, 5] = float("nan")
    deform = (torch.rand((*shape, 3), generator=gen, device=DEV) * 2 - 1) * 0.25
    v, f, gg, gd, w = _loss_grads(grid, deform, 1, normalize)
    v2, f2, gg2, gd2, _ = _loss_grads(grid, deform, 1, normalize)
    assert torch.equal(v.view(torch.int32), v2.view(torch.int32)) and torch.equal(f, f2)
    assert torch.equal(gg.view(torch.int32), gg2.view(torch.int32))
    assert torch.equal(gd.view(torch.int32), gd2.view(torch.int32))

    og = grid.double().requires_grad_(True)
    od = deform.double().requires_grad_(True)
    ov = D.dmc(og, od, iso=0.05, normalize=normalize)[0]
    (ov * w.double() + torch.sin(3 * ov)).sum().backward()
    rel = lambda a, b: float((a.double() - b).norm() / b.norm())
    finite = torch.isfinite(grid)
    assert not gg[~finite].any()
    assert rel(gg[finite], og.grad[finite]) <= 1e-4
    assert rel(gd, od.grad) <= 1e-4


def test_gradient_without_deform_and_unused_outputs():
    grid = D.triposg_field(40, seed=2, device=DEV)
    g = grid.clone().requires_grad_(True)
    v, f = _dmc()(g, normalize=True)
    v[:, 1].sum().backward()
    og = grid.double().requires_grad_(True)
    D.dmc(og)[0][:, 1].sum().backward()
    assert float((g.grad.double() - og.grad).norm() / og.grad.norm()) <= 1e-4


def test_empty_results():
    dmc = _dmc()
    for val in (1.0, -1.0, 0.0):
        for rq in (False, True):
            v, f = dmc(torch.full((5, 6, 7), val, device=DEV), isovalue=0.0, return_quads=rq)
            assert v.shape == (0, 3) and f.shape == (0, 4 if rq else 3)
    grid = torch.full((5, 6, 7), val, device=DEV, requires_grad=True)
    dmc(grid)[0].sum().backward()
    assert grid.grad is not None and not grid.grad.any()
    # a NaN defeats the empty test: an all-below grid is closed by the ring into a box
    grid = -torch.ones((5, 6, 7), device=DEV)
    grid[2, 3, 3] = float("nan")
    v, f = _check(grid, normalize=False)
    assert v.shape[0] > 0 and D.is_oriented_manifold(f.cpu().numpy())
    assert float(v[:, 0].min()) < 0 and float(v[:, 0].max()) > 4


def test_triposg_513_counts_closed_oriented_and_memory():
    grid = D.triposg_field(513, seed=0, device=DEV)
    dmc = _dmc()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    v, f = dmc(grid, normalize=False)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    out = v.numel() * 4 + f.numel() * 4
    assert peak <= out + 64 * 2 ** 20, (peak, out)
    assert (v.shape[0], f.shape[0] // 2) == D.counts(grid)
    fn = f.cpu().numpy()
    assert D.is_oriented_manifold(fn)
    assert D.signed_volume(v.cpu().numpy(), fn[:, ::-1]) > 0


def _logits(n, seed):
    # positive inside, as the VAE decoders return them
    return -D.triposg_field(n, seed=seed, device=DEV) * (n - 1)


def test_hunyuan_dmc_surface_extractor_run():
    # DMCSurfaceExtractor.run (Hunyuan3D 2.0 surface_extractors.py:79-95, 2.1 :127-158): the default extractor of the
    # FlashVDM decoder, on a grid of octree_resolution + 1 points
    octree_resolution = 96
    grid_logit = _logits(octree_resolution + 1, 3)
    dmc = _dmc()
    sdf = (-grid_logit / octree_resolution).to(torch.float32).contiguous()
    verts, faces = dmc(sdf, deform=None, return_quads=False, normalize=True)
    verts = verts - 0.5 * (verts.min(dim=0)[0] + verts.max(dim=0)[0])
    vertices = verts.detach().cpu().numpy()
    faces = faces.detach().cpu().numpy()[:, ::-1]
    assert faces.shape[0] > 0 and D.signed_volume(vertices, faces) > 0


def test_triposg_extraction_tail():
    # TripoSG inference_utils.py:466-472 with the NaN mask its hierarchical decode leaves (:460)
    octree_depth = 7
    octree_resolution = 2 ** octree_depth
    grid_logits = _logits(octree_resolution + 1, 4)
    grid_logits[D.triposg_field(octree_resolution + 1, seed=4, device=DEV, nan_band=True).isnan()] = float("nan")
    bbox_min, bbox_size = np.array([-1.005] * 3), np.array([2.01] * 3)
    dmc = _dmc()
    sdf = (-grid_logits / octree_resolution).to(torch.float32).contiguous()
    vertices, faces = dmc(sdf, deform=None, return_quads=False, normalize=False)
    vertices = vertices.detach().cpu().numpy()
    faces = faces.detach().cpu().numpy()[:, ::-1]
    vertices = vertices / (2 ** octree_depth) * bbox_size + bbox_min
    faces = np.ascontiguousarray(faces)
    assert D.is_oriented_manifold(faces) and D.signed_volume(vertices, faces) > 0


def test_side_stream_and_strided_grid():
    grid = D.triposg_field(33, seed=5, device=DEV)
    ref_v, ref_f = _dmc()(grid)
    s = torch.cuda.Stream()
    t = grid.transpose(0, 2).contiguous().transpose(0, 2)           # same values, non-contiguous
    assert not t.is_contiguous()
    with torch.cuda.stream(s):
        v, f = _dmc()(t)
    s.synchronize()
    assert torch.equal(v, ref_v) and torch.equal(f, ref_f)


def test_errors():
    dmc = _dmc()
    with pytest.raises(TypeError):
        dmc(torch.zeros((4, 4, 4), dtype=torch.float64, device=DEV))
    with pytest.raises(TypeError):
        dmc(torch.zeros((4, 4, 4)))
    with pytest.raises(ValueError):
        dmc(torch.zeros((1, 4, 4), device=DEV), normalize=True)
    with pytest.raises(ValueError):
        dmc(torch.zeros((4, 4, 4), device=DEV), deform=torch.zeros((4, 4, 3), device=DEV))
    one = -torch.ones((1, 4, 4), device=DEV)
    one[0, 3, 3] = 1.0
    v, f = dmc(one, normalize=False)                                    # one layer, closed by the ring
    assert v.shape[0] > 0 and D.is_oriented_manifold(f.cpu().numpy())
