"""StableFast3D's UV texture baker on the GPU (gs_b200.uv_bake, the slangtorch shim): bit-exact against the numpy oracle
on the golden SF3D atlases, synthetic soups and the adversarial set through every queue, against the reference's own
kernels (the oracle/_ref build) where it exists, the launched-region rule, face ids above 2^24, TextureBaker's call
sequence, and run-to-run bits."""
import hashlib
import importlib.util
import os

import numpy as np
import pytest
import torch

from oracle import build_ref_sf3d
from oracle import uvbake_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_sf3d_baker.npz")
DEV = torch.device("cuda:0")
SENT = -7.25


def _mk():
    spec = importlib.util.spec_from_file_location("make_golden_sf3d_baker",
                                                  os.path.join(ROOT, "tests", "golden", "make_golden_sf3d_baker.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


def _ub():
    from gs_b200 import uv_bake
    return uv_bake


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _bits(t):
    return t.detach().contiguous().cpu().numpy().view(np.uint32)


def _bake(uv, faces, res, rows=None, cols=None, counts=False):
    rows = res if rows is None else rows
    cols = res if cols is None else cols
    out = torch.full((res, res, 4), SENT, device=DEV)
    return _ub().rasterize_into(_t(uv), _t(faces), out, rows, cols, counts=counts)


def _oracle(uv, faces, res, rows=None, cols=None):
    return O.rasterize(uv, faces, res, rows, cols, out=np.full((res, res, 4), SENT, np.float32))


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).digest()


# ---- golden SF3D atlases (the reference's own bakes) ----------------------------------------------------------------
def _golden_cases():
    if not os.path.isfile(GOLDEN):
        return []
    return [(n, r) for n in _mk().MESHES for r in _mk().RESOLUTIONS]


@pytest.mark.parametrize("name,res", _golden_cases())
def test_golden_bit_exact(name, res):
    mk = _mk()
    z = dict(np.load(GOLDEN))
    uv, faces, pos, nrm = (None if a is None else _t(a) for a in mk.soup(z, name))
    key = f"{name}/{res}"
    n = (res // 16) * 16
    rast = _ub().rasterize_into(uv, faces, torch.full((res, res, 4), SENT, device=DEV), n, n)
    if f"{key}/rast" in z:
        assert np.array_equal(_bits(rast), z[f"{key}/rast"])
    assert _sha(rast) == z[f"{key}/rast_sha256"].tobytes()
    for nm, attr in (("pos_bake", pos), ("nrm_bake", nrm)):
        if attr is None:
            continue
        got = _ub().interpolate_into(attr, rast, faces, torch.full((res, res, 3), SENT, device=DEV), n, n)
        assert _sha(got) == z[f"{key}/{nm}_sha256"].tobytes(), nm


def test_texture_baker_sequence_through_slangtorch():
    """sf3d/texture_baker.py's TextureBaker, restated call for call over the shim's module (res % 16 != 0 included)."""
    import slangtorch
    mod = slangtorch.TextureBakerModule()
    uv, faces = O.soup(5000, 3)
    pos = np.random.default_rng(3).standard_normal((uv.shape[0], 3)).astype(np.float32)
    for res in (200, 256):
        g = res // 16
        rast = torch.empty(res, res, 4, device=DEV)
        rast[:] = SENT                                      # what torch.empty happened to hold
        mod.bake_uv(uv=_t(uv), indices=_t(faces).to(torch.int32), output=rast).launchRaw(
            blockSize=(16, 16, 1), gridSize=(g, g, 1))
        mask = rast[..., -1] >= 0
        pos_bake = torch.zeros(res, res, 3, device=DEV)
        mod.interpolate(attr=_t(pos), indices=_t(faces), rast=rast, output=pos_bake).launchRaw(
            blockSize=(16, 16, 1), gridSize=(g, g, 1))
        want = _oracle(uv, faces, res, g * 16, g * 16)
        assert np.array_equal(_bits(rast), want.view(np.uint32))
        wp = O.interpolate(pos, want, faces, g * 16, g * 16)
        assert np.array_equal(_bits(pos_bake), wp.view(np.uint32))
        assert int(mask.sum()) > 0


# ---- synthetic soups and the adversarial set against the oracle ------------------------------------------------------
@pytest.mark.parametrize("F,res,seed", [(20000, 512, 1), (60000, 1000, 2), (3000, 97, 3)])
def test_soup_bit_exact(F, res, seed):
    uv, faces = O.soup(F, seed)
    got = _bake(uv, faces, res)
    assert np.array_equal(_bits(got), _oracle(uv, faces, res).view(np.uint32))


@pytest.mark.parametrize("name", sorted(O.adversarial(0)))
def test_adversarial_bit_exact(name):
    uv, faces, res = O.adversarial(0)[name]
    got = _bake(uv, faces, res)
    assert np.array_equal(_bits(got), O.rasterize(uv, faces, res, mode="brute").view(np.uint32))


@pytest.mark.parametrize("name", sorted(O.queue_cases(0)))
def test_queue_cases_bit_exact_and_counts(name):
    uv, faces, res = O.queue_cases(0)[name]
    got, (warp, cta, whole) = _bake(uv, faces, res, counts=True)
    thread_o, warp_o, cta_o, whole_o = O.queue_counts(uv, faces, res)
    assert (warp, cta, whole) == (warp_o, cta_o, whole_o)
    F = faces.shape[0]
    want = {"thread": thread_o == F, "warp": warp > F // 2, "cta_split": 0 < cta <= 132 * 8,
            "cta_whole": cta > 132 * 8 and whole == 0, "whole_texture": whole == F}[name]
    assert want, (name, thread_o, warp, cta, whole)
    assert np.array_equal(_bits(got), _oracle(uv, faces, res).view(np.uint32))


def test_region_leaves_unlaunched_texels():
    uv, faces = O.soup(4000, 5)
    for rows, cols in ((96, 96), (37, 100), (0, 50), (100, 100), (500, 500)):
        got = _bake(uv, faces, 100, rows, cols)
        r, c = min(rows, 100), min(cols, 100)
        assert np.array_equal(_bits(got), _oracle(uv, faces, 100, r, c).view(np.uint32))
        g = got.cpu()
        assert (g[r:] == SENT).all() and (g[:, c:] == SENT).all()


def test_face_ids_above_2_24():
    """2^24 + 64 faces, all degenerate (dropped) but the last 64: the winner's id rounds as float(i) does."""
    uv, faces = O.soup(64, 7)
    F0 = (1 << 24) + 64
    big = torch.zeros(F0, 3, dtype=torch.int32, device=DEV)
    big[F0 - 64:] = _t(faces)
    got = _ub().rasterize_into(_t(uv), big, torch.full((64, 64, 4), SENT, device=DEV), 64, 64)
    want = _oracle(uv, faces, 64)
    hit = want[..., 3] >= 0
    want[..., 3] = np.where(hit, (want[..., 3].astype(np.int64) + F0 - 64).astype(np.float32), want[..., 3])
    assert hit.any()
    assert np.array_equal(_bits(got), want.view(np.uint32))
    assert (got[..., 3][torch.from_numpy(hit).to(DEV)] >= 2.0 ** 24).all()


def test_out_of_range_ids_and_int64_faces():
    uv, faces = O.soup(500, 8)
    bad = faces.copy()
    bad[::7, 1] = uv.shape[0] + 3
    bad[3::11, 2] = -2
    got = _bake(uv, bad.astype(np.int64), 64)
    assert np.array_equal(_bits(got), _oracle(uv, bad, 64).view(np.uint32))
    attr = np.random.default_rng(0).standard_normal((uv.shape[0], 3)).astype(np.float32)
    rast = got.clone()
    rast[0, :8, 3] = torch.tensor([float("nan"), -0.5, 1e10, -1e10, 499.9, 500.0, float("inf"), 2.0 ** 31])
    out = _ub().interpolate_into(_t(attr), rast, _t(bad), torch.full((64, 64, 3), SENT, device=DEV), 64, 64)
    want = O.interpolate(attr, rast.cpu().numpy(), bad)
    assert np.array_equal(_bits(out), want.view(np.uint32))


def test_run_to_run_bits_and_streams():
    uv, faces = O.soup(30000, 9)
    a = _bake(uv, faces, 1024)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        b = _bake(uv, faces, 1024)
    s.synchronize()
    assert np.array_equal(_bits(a), _bits(b))


def test_errors():
    ub = _ub()
    uv = torch.rand(6, 2, device=DEV)
    f = torch.arange(6, dtype=torch.int32, device=DEV).reshape(2, 3)
    with pytest.raises(NotImplementedError):
        ub.rasterize_into(uv, f, torch.empty(16, 8, 4, device=DEV), 16, 8)
    with pytest.raises(ValueError):
        ub.rasterize_into(uv, f, torch.empty(16, 16, 4, device=DEV).transpose(0, 1), 16, 16)
    with pytest.raises(TypeError):
        ub.rasterize_into(uv.double(), f, torch.empty(16, 16, 4, device=DEV), 16, 16)


# ---- the reference's own kernels (oracle/_ref) ----------------------------------------------------------------------
def _ref():
    lib = build_ref_sf3d.load()
    if lib is None:
        pytest.skip("oracle/_ref has no SF3D reference build (no ComfyUI-3D-Pack checkout was found: see "
                    "oracle/build_ref_sf3d.py)")
    return lib


def _ref_bake(lib, uv, faces, res, rows, cols):
    out = torch.full((res, res, 4), SENT, device=DEV)
    assert lib.sf3d_ref_bake_uv(uv.data_ptr(), uv.shape[0], faces.data_ptr(), faces.shape[0], out.data_ptr(), res, res,
                                16, 16, rows // 16, cols // 16, torch.cuda.current_stream().cuda_stream) == 0
    return out


def _ref_interp(lib, attr, faces, rast, rows, cols):
    res = rast.shape[0]
    out = torch.full((res, res, 3), SENT, device=DEV)
    assert lib.sf3d_ref_interpolate(attr.data_ptr(), attr.shape[0], faces.data_ptr(), faces.shape[0], rast.data_ptr(),
                                    out.data_ptr(), res, res, 16, 16, rows // 16, cols // 16,
                                    torch.cuda.current_stream().cuda_stream) == 0
    return out


@pytest.mark.parametrize("F,res,seed", [(100000, 2048, 1), (20000, 1000, 2), (100000, 1024, 3)])
def test_reference_build_bit_exact(F, res, seed):
    lib = _ref()
    uv, faces = O.soup(F, seed)
    rng = np.random.default_rng(seed)
    pos = _t(rng.standard_normal((uv.shape[0], 3)).astype(np.float32))
    nrm = torch.nn.functional.normalize(_t(rng.standard_normal((uv.shape[0], 3)).astype(np.float32)), dim=-1)
    uv, faces = _t(uv), _t(faces)
    n = (res // 16) * 16
    ref = _ref_bake(lib, uv, faces, res, n, n)
    got = _ub().rasterize_into(uv, faces, torch.full((res, res, 4), SENT, device=DEV), n, n)
    assert np.array_equal(_bits(got), _bits(ref))
    for attr in (pos, nrm):
        r = _ref_interp(lib, attr, faces, ref, n, n)
        g = _ub().interpolate_into(attr, got, faces, torch.full((res, res, 3), SENT, device=DEV), n, n)
        assert np.array_equal(_bits(g), _bits(r))


@pytest.mark.parametrize("name", sorted(O.adversarial(0)) + sorted(O.queue_cases(0)))
def test_reference_build_adversarial(name):
    lib = _ref()
    cases = {**O.adversarial(0), **O.queue_cases(0)}
    uv, faces, res = cases[name]
    n = (res // 16) * 16
    ref = _ref_bake(lib, _t(uv), _t(faces), res, n, n)
    got = _ub().rasterize_into(_t(uv), _t(faces), torch.full((res, res, 4), SENT, device=DEV), n, n)
    assert np.array_equal(_bits(got), _bits(ref))
