"""CPU tests of the dual-marching-cubes oracle (oracle/dmc_oracle.py) and the `diso` import shim.

The oracle is what the GPU kernels (csrc/ngp_dmc.cu) are held to, so its rules are anchored here on cases worked by
hand, on fields whose exact surface is known, on mesh topology, and on autograd against finite differences."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import dmc_oracle as D


def _mesh_ok(grid, iso=0.0, genus=0):
    v, f, _ = D.dmc(grid, iso=iso, normalize=False)
    f = f.numpy()
    assert D.is_oriented_manifold(f)
    assert D.euler_characteristic(len(v), f) == 2 - 2 * genus
    return v.numpy(), f


def test_one_corner_below_gives_the_hand_computed_box():
    # a single below sample at (0,0,0) of a 2x2x2 grid: its 6 edges (3 to the ring) cross at +-0.5, and each of the 8
    # cubes around it averages its 3 crossings to (+-1/6, +-1/6, +-1/6), cubes in padded linear order
    g = torch.ones((2, 2, 2), dtype=torch.float64)
    g[0, 0, 0] = -1
    v, q, _ = D.dmc(g, return_quads=True, normalize=True)
    s = lambda b: 1 / 6 if b else -1 / 6
    want = torch.tensor([[s(i), s(j), s(k)] for i in (0, 1) for j in (0, 1) for k in (0, 1)], dtype=torch.float64)
    assert torch.allclose(v, want, rtol=0, atol=1e-15)
    assert q.shape == (6, 4)
    tris = D.dmc(g, normalize=True)[1].numpy()
    assert tris.shape == (12, 3) and D.is_oriented_manifold(tris) and D.euler_characteristic(8, tris) == 2
    # triangles run counter-clockwise seen from the below side: normals point into the below region
    assert D.signed_volume(v.numpy(), tris) < 0 < D.signed_volume(v.numpy(), tris[:, ::-1])
    # first quad: the x edge from the ring point (-1,0,0), above, to (0,0,0), below; its cubes (db, dc) over (y, z)
    # from the lowest: (1,1), (0,1), (0,0), (1,0) -> padded cubes (0,0,0), (0,1,0), (0,1,1), (0,0,1)
    assert q[0].tolist() == [0, 2, 3, 1]


def test_tilted_plane_vertices_lie_on_the_plane():
    n = torch.tensor([0.3, -0.5, 0.8], dtype=torch.float64)
    X, Y, Z = 9, 11, 13
    idx = torch.stack(torch.meshgrid(*[torch.arange(d, dtype=torch.float64) for d in (X, Y, Z)], indexing="ij"), -1)
    g = idx @ n - 1.7
    v, f, _ = D.dmc(g, iso=0.25, normalize=False)
    # vertices of cubes clear of the ring (strictly inside the unpadded box) average crossings of the linear field
    inner = ((v > 0) & (v < torch.tensor([X - 1, Y - 1, Z - 1], dtype=torch.float64))).all(-1)
    assert int(inner.sum()) > 50
    assert float((v[inner] @ n - 1.7 - 0.25).abs().max()) < 1e-12


def test_sphere_is_closed_and_oriented():
    n = 24
    idx = np.indices((n, n, n)).transpose(1, 2, 3, 0).astype(np.float64)
    g = torch.from_numpy(np.linalg.norm(idx - [11.3, 12.1, 11.7], axis=-1) - 8.2)
    v, f = _mesh_ok(g, genus=0)
    assert D.signed_volume(v, f[:, ::-1]) == pytest.approx(4 / 3 * np.pi * 8.2 ** 3, rel=0.02)


def test_torus_is_closed_with_euler_characteristic_zero():
    n = 32
    p = np.indices((n, n, n)).transpose(1, 2, 3, 0).astype(np.float64) - [15.5, 15.2, 15.8]
    g = torch.from_numpy(np.hypot(np.hypot(p[..., 0], p[..., 1]) - 9.0, p[..., 2]) - 3.5)
    _mesh_ok(g, genus=1)


def test_border_cut_surface_is_closed_by_the_ring():
    n = 16
    idx = np.indices((n, n, n)).transpose(1, 2, 3, 0).astype(np.float64)
    g = torch.from_numpy(np.linalg.norm(idx - [0.3, 7.4, 15.2], axis=-1) - 6.5)
    _mesh_ok(g, genus=0)


def test_oracle_gradients_match_finite_differences():
    gen = torch.Generator().manual_seed(3)
    g = (torch.rand((5, 6, 7), generator=gen, dtype=torch.float64) * 2 - 1).requires_grad_(True)
    d = ((torch.rand((5, 6, 7, 3), generator=gen, dtype=torch.float64) * 2 - 1) * 0.2).requires_grad_(True)
    assert min(float(g.detach().abs().min()), 1.0) > 1e-4       # no sample so near iso that eps changes the case
    assert torch.autograd.gradcheck(lambda a, b: D.dmc(a, b, iso=0.0, normalize=True)[0], (g, d), eps=1e-6, atol=1e-6,
                                    rtol=1e-5)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_counts_agree_with_the_full_oracle(seed):
    gen = torch.Generator().manual_seed(seed)
    g = torch.rand((13, 9, 17), generator=gen) * 2 - 1
    g[torch.rand(g.shape, generator=gen) < 0.03] = float("nan")
    g[torch.rand(g.shape, generator=gen) < 0.01] = float("inf")
    v, _, info = D.dmc(g, iso=0.1)
    assert D.counts(g, iso=0.1) == (v.shape[0], info["quads"].shape[0])
    f = D.triposg_field(64, seed=seed, nan_band=True)
    assert torch.isnan(f).any()
    v, _, info = D.dmc(f, normalize=False)
    assert D.counts(f) == (v.shape[0], info["quads"].shape[0]) and v.shape[0] > 0
    assert not torch.isnan(v).any()


def test_empty_rule():
    for g in (torch.ones((4, 4, 4)), -torch.ones((4, 4, 4)), torch.zeros((4, 4, 4))):
        v, f, _ = D.dmc(g)
        assert v.shape == (0, 3) and f.shape == (0, 3) and D.counts(g) == (0, 0)
    # a NaN defeats the test; all-below is then closed by the ring into a box around the finite cubes
    g = -torch.ones((4, 5, 6))
    g[2, 2, 2] = float("nan")
    v, f, _ = D.dmc(g, normalize=False)
    assert v.shape[0] > 0 and D.is_oriented_manifold(f.numpy())


def test_diso_import_resolves_to_the_shim_and_refuses_what_it_cannot_run():
    import diso
    assert os.path.realpath(diso.__file__).startswith(os.path.realpath(os.path.join(ROOT, "comfyui-3d-pack_b200")))
    with pytest.raises(NotImplementedError):
        diso.DiffDMC(dtype=torch.float64)
    with pytest.raises(NotImplementedError):
        diso.DiffMC(dtype=torch.float32)
    dmc = diso.DiffDMC(dtype=torch.float32).to("cpu")
    assert list(dmc.parameters()) == []
    with pytest.raises(TypeError):
        dmc(torch.zeros((4, 4, 4)))
