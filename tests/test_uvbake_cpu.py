"""StableFast3D's UV texture baker, CPU side: the numpy oracle against the reference's own bakes (the golden fixture),
its exact fp32 FMA against fractions, the candidate-box rule against brute force on adversarial soups, the slangtorch
shim's refusals, and the C ABI."""
import os
from fractions import Fraction

import numpy as np
import pytest

from oracle import uvbake_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_sf3d_baker.npz")


def _golden():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_sf3d_baker",
                                                  os.path.join(ROOT, "tests", "golden", "make_golden_sf3d_baker.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk, dict(np.load(GOLDEN))


def _round_f32(x):
    """Fraction -> nearest fp32, ties to even (finite range)."""
    r = np.float32(float(x))
    best = None
    for c in (np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))):
        if not np.isfinite(c):
            continue
        d = abs(Fraction(float(c)) - x)
        key = (d, int(np.array(c, np.float32).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return np.float32(best[1])


def test_fma32_exact_against_fractions():
    rng = np.random.default_rng(0)
    n = 4000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(n) * 2.0 ** -rng.integers(1, 60, n))).astype(np.float32)
    # midpoint cases: c chosen so that a*b + c sits next to a halfway point of fp32, where float64 rounds twice
    half = (np.float32(1) + np.float32(2.0 ** -23)).astype(np.float32)
    a = np.concatenate([a, np.full(8, half, np.float32), np.float32([0.5, -0.0, 3.0, 1e-20])])
    b = np.concatenate([b, np.full(8, half, np.float32), np.float32([-0.0, 5.0, -7.0, 1e-20])])
    c = np.concatenate([c, np.float32([2.0 ** -48, -2.0 ** -48, 2.0 ** -70, -2.0 ** -70, 0, -1, 1, 2.0 ** -24]),
                        np.float32([0.0, 0.0, 21.0, 0.0])])
    got = O.fma32(a, b, c)
    for x, y, z, g in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        want = _round_f32(exact)
        if exact == 0:                      # the sign of an exact zero: +0 unless both addends are -0
            want = np.float32(-0.0) if (np.signbit(np.float32(x) * np.float32(y)) and np.signbit(z)) else np.float32(0)
        assert np.float32(g).view(np.uint32) == want.view(np.uint32), (x, y, z, g, want)


def test_dot_zero_product_is_positive_zero():
    # the reference's dot starts from +0, so (-0) + (-0) never appears
    assert not np.signbit(O.dot2(np.float32(-0.0), np.float32(0.0), np.float32(1.0), np.float32(-0.0)))


@pytest.mark.parametrize("name", sorted(O.adversarial(0)))
def test_box_rule_equals_brute_force(name):
    uv, faces, res = O.adversarial(0)[name]
    a = O.rasterize(uv, faces, res, mode="brute")
    b = O.rasterize(uv, faces, res, mode="box")
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("seed", [1, 2])
def test_box_rule_equals_brute_force_region_and_soup(seed):
    uv, faces = O.soup(600, seed)
    for rows, cols in ((48, 48), (37, 50)):
        a = O.rasterize(uv, faces, 50, rows, cols, mode="brute")
        b = O.rasterize(uv, faces, 50, rows, cols, mode="box")
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        assert np.isnan(a[rows:]).all() and np.isnan(a[:, cols:]).all()


def test_queue_cases_reach_their_queue():
    for name, (uv, faces, res) in O.queue_cases(0).items():
        thread, warp, cta, whole = O.queue_counts(uv, faces, res)
        F = faces.shape[0]
        if name == "thread":
            assert thread == F
        elif name == "warp":
            assert warp > F // 2
        elif name == "cta_split":
            assert 0 < cta <= 132 * 8
        elif name == "cta_whole":
            assert cta > 132 * 8 and whole == 0
        elif name == "whole_texture":
            assert whole == F


def test_oracle_equals_golden_bits():
    mk, z = _golden()
    sentinel = z["sentinel"].view(np.float32)[0]
    import hashlib
    for name in mk.MESHES:
        uv, faces, pos, nrm = mk.soup(z, name)
        for res in mk.RESOLUTIONS:
            key = f"{name}/{res}"
            n = (res // 16) * 16
            rast = O.rasterize(uv, faces, res, n, n, out=np.full((res, res, 4), sentinel, np.float32))
            if f"{key}/rast" in z:
                assert np.array_equal(rast.view(np.uint32), z[f"{key}/rast"]), key
            assert hashlib.sha256(rast.tobytes()).digest() == z[f"{key}/rast_sha256"].tobytes(), key
            for nm, attr in (("pos_bake", pos), ("nrm_bake", nrm)):
                if attr is None:
                    continue
                got = O.interpolate(attr, rast, faces, n, n, out=np.full((res, res, 3), sentinel, np.float32))
                if f"{key}/{nm}" in z:
                    assert np.array_equal(got.view(np.uint32), z[f"{key}/{nm}"]), (key, nm)
                assert hashlib.sha256(got.tobytes()).digest() == z[f"{key}/{nm}_sha256"].tobytes(), (key, nm)


def test_interpolate_oracle_edges():
    attr = np.arange(12, dtype=np.float32).reshape(4, 3)
    faces = np.array([[0, 1, 2], [1, 2, 3], [0, 9, 1]], np.int32)
    rast = np.zeros((1, 6, 4), np.float32)
    rast[0, :, 3] = [0.9, -0.5, np.nan, 2.0, -1.0, 3e9]
    rast[0, :, :3] = [0.25, 0.5, 0.25]
    out = O.interpolate(attr, rast, faces)
    # 0.9 and -0.5 and NaN truncate to face 0; face 2 has an out-of-range vertex; -1 and 3e9 are out of range
    want0 = O.fma32(np.float32(0.25), attr[2], O.fma32(np.float32(0.25), attr[0], np.float32(0.5) * attr[1]))
    for k in (0, 1, 2):
        assert np.array_equal(out[0, k], want0)
    assert (out[0, 3:] == 0).all()


def test_slangtorch_shim_hash_and_refusals(tmp_path):
    slangtorch = pytest.importorskip("slangtorch")
    other = tmp_path / "other.slang"
    other.write_text("// not the texture baker\n")
    with pytest.raises(NotImplementedError, match="other.slang"):
        slangtorch.loadModule(str(other))
    with pytest.raises(NotImplementedError):
        slangtorch.loadModule(str(tmp_path / "missing.slang"))
    # the CRLF form of a file hashes as its LF form
    crlf = tmp_path / "crlf.slang"
    crlf.write_bytes(b"a\r\nb\r\n")
    lf = tmp_path / "lf.slang"
    lf.write_bytes(b"a\nb\n")
    assert slangtorch.file_sha256(str(crlf)) == slangtorch.file_sha256(str(lf))


def test_slangtorch_shim_reference_hash():
    slangtorch = pytest.importorskip("slangtorch")
    from oracle import build_ref_sf3d
    src = build_ref_sf3d.source()
    if src is None:
        pytest.skip("no ComfyUI-3D-Pack checkout found (see oracle/build_ref_sf3d.py)")
    path = os.path.join(src.split("/.slangtorch_cache/")[0], "texture_baker.slang")
    assert slangtorch.file_sha256(path) == slangtorch.TEXTURE_BAKER_SHA256
    mod = slangtorch.loadModule(path)
    assert hasattr(mod, "bake_uv") and hasattr(mod, "interpolate")


def test_cpu_tensors_raise():
    import torch
    from gs_b200 import uv_bake
    uv = torch.rand(6, 2)
    faces = torch.arange(6, dtype=torch.int32).reshape(2, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        uv_bake.rasterize(uv, faces, 16)
    with pytest.raises(RuntimeError, match="CUDA"):
        uv_bake.interpolate(torch.rand(6, 3), torch.zeros(16, 16, 4), faces)
    import slangtorch
    launch = slangtorch.TextureBakerModule().bake_uv(uv=uv, indices=faces, output=torch.empty(16, 16, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        launch.launchRaw(blockSize=(16, 16, 1), gridSize=(1, 1, 1))


def test_abi_scratch_bytes():
    from gs_b200 import _lib
    sb = _lib.lib.dr_b200_uvbake_scratch_bytes
    assert sb(0, 16) == 256 + 16 * 16 * 4
    assert sb(1000, 1024) == 256 + 1024 * 1024 * 4 + 8000
    assert sb(10 ** 6, 8192) == 256 + 8192 * 8192 * 4 + 8 * 10 ** 6
    assert sb(-1, 16) == 0 and sb(5, 0) == 0 and sb(5, (1 << 15) + 1) == 0
