"""Marching cubes on the H100 (csrc/ngp_mcubes.cu via gs_b200.isosurface and the `mcubes` shim): bit-identical to
the numpy oracle (oracle/mc_oracle.py) in vertex fp32 bits, triangle indices and both orders."""
import numpy as np
import pytest
import torch

from conftest import ROOT  # noqa: F401
from oracle import mc_oracle as M

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _gpu(vol, iso):
    from gs_b200.isosurface import marching_cubes
    v, t = marching_cubes(torch.from_numpy(np.ascontiguousarray(vol)).to(DEV), iso)
    assert v.dtype == torch.float32 and t.dtype == torch.int32 and v.device == DEV and t.device == DEV
    return v.cpu().numpy(), t.cpu().numpy()


def _assert_matches_oracle(vol, iso):
    gv, gt = _gpu(vol, iso)
    ov, ot = M.marching_cubes(vol, iso)
    assert gv.shape == ov.shape and gt.shape == ot.shape, (gv.shape, ov.shape, gt.shape, ot.shape)
    assert np.array_equal(gv.view(np.uint32), ov.view(np.uint32))
    assert np.array_equal(gt, ot)
    return gv, gt


def test_every_configuration_matches_the_oracle():
    rng = np.random.default_rng(0)
    for cube in range(256):
        bits = np.array([(cube >> i) & 1 for i in range(8)], dtype=bool)
        vals = np.where(bits, rng.uniform(0.05, 1.0, 8), rng.uniform(-1.0, -0.05, 8)).astype(np.float32)
        vol = np.empty((2, 2, 2), np.float32)
        for i in range(8):
            vol[i & 1, (i >> 1) & 1, i >> 2] = vals[i]
        v, t = _assert_matches_oracle(vol, 0.0)
        assert len(t) == M.load_table()[0][cube]


@pytest.mark.parametrize("seed,shape,iso", [(0, (17, 33, 65), 0.1), (1, (40, 40, 40), 0.0), (2, (5, 70, 3), -0.2),
                                             (3, (2, 2, 2), 0.0), (4, (65, 9, 130), 0.3)])
def test_random_fields_match_the_oracle(seed, shape, iso):
    vol = np.random.default_rng(seed).uniform(-1, 1, shape).astype(np.float32)
    _assert_matches_oracle(vol, iso)


def test_sphere_128_matches_the_oracle_and_is_closed():
    n, r, c = 128, 50.3, np.array([63.7, 64.2, 63.9])
    g = np.indices((n, n, n)).astype(np.float64).transpose(1, 2, 3, 0)
    vol = (r - np.linalg.norm(g - c, axis=-1)).astype(np.float32)
    v, t = _assert_matches_oracle(vol, 0.0)
    assert M.is_oriented_manifold(t) and M.euler_characteristic(len(v), t) == 2


def test_blob_density_256_matches_the_oracle_in_full():
    vol = M.blob_density(256, seed=0).numpy()
    v, t = _assert_matches_oracle(vol, 10.0)
    assert len(t) > 100_000
    assert M.is_closed_oriented(t)


def test_two_runs_are_bit_identical():
    vol = M.blob_density(96, seed=1).numpy()
    a, b = _gpu(vol, 10.0), _gpu(vol, 10.0)
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])


def test_runs_on_the_current_stream():
    from gs_b200.isosurface import marching_cubes
    vol = torch.from_numpy(M.blob_density(64, seed=2).numpy()).to(DEV)
    ref = marching_cubes(vol, 10.0)
    s = torch.cuda.Stream(device=DEV)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        got = marching_cubes(vol, 10.0)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(ref[0], got[0]) and torch.equal(ref[1], got[1])


@pytest.mark.parametrize("shape,fill", [((16, 16, 16), -1.0), ((16, 16, 16), 1.0), ((1, 16, 16), -1.0),
                                        ((16, 1, 16), 1.0), ((16, 16, 1), 0.0), ((0, 4, 4), 0.0)])
def test_empty_results(shape, fill):
    vol = np.full(shape, fill, np.float32)
    if fill == 0.0 and shape[0]:
        vol[:, ::2] = 1.0                         # a size-1 axis with crossings along the others still has no cell
    v, t = _gpu(vol, 0.5)
    assert v.shape == (0, 3) and t.shape == (0, 3)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_sample_raises(bad):
    vol = np.random.default_rng(5).uniform(-1, 1, (20, 21, 22)).astype(np.float32)
    vol[7, 13, 21] = bad
    with pytest.raises(RuntimeError, match="non-finite"):
        _gpu(vol, 0.0)
    _gpu(np.nan_to_num(vol, nan=0.0, posinf=1.0, neginf=-1.0), 0.0)   # the library is usable after the error


def test_numpy_shim_equals_the_device_result():
    import mcubes
    vol64 = M.blob_density(80, seed=3).numpy().astype(np.float64)
    v, t = mcubes.marching_cubes(vol64, 10)
    dv, dt = _gpu(vol64.astype(np.float32), 10.0)
    assert v.dtype == mcubes.VERTEX_DTYPE and t.dtype == mcubes.TRIANGLE_DTYPE
    assert np.array_equal(v, dv.astype(np.float64)) and np.array_equal(t, dt.astype(np.uint64))
    vi, ti = mcubes.marching_cubes((vol64 * 4).astype(np.int16), 40)          # any real dtype is cast to fp32
    di = _gpu((vol64 * 4).astype(np.int16).astype(np.float32), 40.0)
    assert np.array_equal(vi, di[0].astype(np.float64)) and np.array_equal(ti, di[1].astype(np.uint64))


def test_reference_call_form_gives_a_closed_outward_mesh():
    """mesh_processer/mesh_utils.py:493-514: density sampled in S^3 chunks on a linspace grid, then
    `vertices, triangles = marching_cubes(sigmas, density_thresh)` and the rescale to [-1, 1]."""
    from mcubes import marching_cubes
    grid_size, S, density_thresh = 128, 64, 10
    rng = np.random.default_rng(7)
    centres = torch.tensor(rng.uniform(-0.4, 0.4, (5, 3)), dtype=torch.float32, device=DEV)
    widths = torch.tensor(rng.uniform(0.1, 0.25, (5, 3)), dtype=torch.float32, device=DEV)

    def get_density_func(pts):
        q = (pts.to(DEV)[:, None, :] - centres) / widths
        return (40.0 * torch.exp(-0.5 * (q * q).sum(-1))).sum(-1, keepdim=True)

    sigmas = np.zeros([grid_size, grid_size, grid_size], dtype=np.float32)
    X = torch.linspace(-1, 1, grid_size).split(S)
    Y = torch.linspace(-1, 1, grid_size).split(S)
    Z = torch.linspace(-1, 1, grid_size).split(S)
    for xi, xs in enumerate(X):
        for yi, ys in enumerate(Y):
            for zi, zs in enumerate(Z):
                xx, yy, zz = torch.meshgrid(xs, ys, zs, indexing='ij')
                pts = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1), zz.reshape(-1, 1)], dim=-1)
                val = get_density_func(pts)
                sigmas[xi * S: xi * S + len(xs), yi * S: yi * S + len(ys), zi * S: zi * S + len(zs)] = \
                    val.reshape(len(xs), len(ys), len(zs)).detach().cpu().numpy()
    vertices, triangles = marching_cubes(sigmas, density_thresh)
    vertices = vertices / (grid_size - 1.0) * 2 - 1
    vertices = vertices.astype(np.float32)
    triangles = triangles.astype(np.int32)
    assert len(triangles) > 1000 and np.abs(vertices).max() <= 1.0
    assert M.is_closed_oriented(triangles)
    # outward normals: the signed volume is positive and close to the volume of the above-threshold samples
    cell = (2.0 / (grid_size - 1)) ** 3
    vol = M.signed_volume(vertices, triangles)
    assert vol > 0 and abs(vol / (float((sigmas > density_thresh).sum()) * cell) - 1) < 0.05
