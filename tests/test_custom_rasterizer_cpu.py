"""Hunyuan3D's custom_rasterizer drop-in, without a GPU: the numpy oracle against the reference's own outputs (the
golden fixture, and the reference's CPU path when oracle/_ref holds its build), the two import shims and the C ABI."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import build_ref
from oracle import cr_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_custom_rasterizer.npz")
RASTER, INTERP = O.golden_cases(GOLDEN)


def _same(fi, b, case):
    if case["digest"] is not None:
        return O.digest(fi, b) == case["digest"] and int((fi != 0).sum()) == case["covered"]
    return np.array_equal(fi, case["findices"]) and np.array_equal(b.view(np.uint32), case["bary"].view(np.uint32))


@pytest.mark.parametrize("name", sorted(RASTER))
def test_oracle_matches_golden_rasterize(name):
    c = RASTER[name]
    H, W = c["hw"]
    fi, b = O.rasterize(c["pos"], c["tri"], W, H, c["depth"])
    assert _same(fi, b, c)


@pytest.mark.parametrize("name", sorted(INTERP))
def test_oracle_matches_golden_interpolate(name):
    c = INTERP[name]
    r = RASTER[c["src"]]
    H, W = r["hw"]
    fi, b = O.rasterize(r["pos"], r["tri"], W, H, r["depth"])
    out = O.interpolate(c["col"], fi.astype(np.float32) if c["fp32_ids"] else fi, b, r["tri"])
    if c["out_digest"] is not None:
        assert hashlib.sha256(out.astype(np.float32).tobytes()).hexdigest() == c["out_digest"]
    else:
        assert np.array_equal(out.view(np.uint32), c["out"].view(np.uint32))


def test_golden_covers_the_edge_cases():
    assert RASTER["no_faces"]["tri"].shape == (0, 3)
    assert RASTER["depth_prior"]["depth"] is not None
    assert (RASTER["w_negative"]["pos"][:, 3] < 0).any() and RASTER["w_negative"]["findices"].any()
    assert min(RASTER["line_1x37"]["hw"]) == 1 and min(RASTER["line_29x1"]["hw"]) == 1
    assert RASTER["view_persp_383x257"]["covered"] > 0 and RASTER["uv_256"]["covered"] > 0
    assert any(c["fp32_ids"] for c in INTERP.values()) and any(not c["fp32_ids"] for c in INTERP.values())
    assert any(c["tri_i64"] for c in INTERP.values()) and any(not c["tri_i64"] for c in INTERP.values())
    eq = RASTER["equal_depth"]["findices"]          # faces 0 and 2 are the same triangle: 2 never wins
    assert (eq == 1).any() and not (eq == 3).any()


def _ref_cpu():
    mod = build_ref.load("nofma")
    if mod is None:
        pytest.skip("oracle/_ref has no reference build (no ComfyUI-3D-Pack checkout was found: see oracle/build_ref.py)")
    return mod


@pytest.mark.parametrize("seed", range(8))
def test_oracle_matches_reference_cpu_sweep(seed):
    ref = _ref_cpu()
    rng = np.random.default_rng(100 + seed)
    N, NF = 200, 400
    V = np.concatenate([rng.uniform(-1.3, 1.3, (N, 3)), rng.uniform(0.2, 1.5, (N, 1))], 1).astype(np.float32)
    V[: seed % 4, 3] *= -1                                         # some w < 0
    if seed % 3 == 0:                                              # vertices on pixel centres, shared by many faces
        V[:, :2] = np.round(V[:, :2] * 8) / 8
    F = rng.integers(0, N, (NF, 3)).astype(np.int32)
    W, H = [(48, 36), (37, 53), (1, 9), (64, 64)][seed % 4]       # W = 1: every face has zero area, nothing covered
    D = rng.uniform(-1, 1, (H, W)).astype(np.float32) if seed % 2 else None
    fi, b = ref.rasterize_image(torch.from_numpy(V), torch.from_numpy(F), torch.from_numpy(D) if D is not None
                                else torch.zeros(0), W, H, 1e-6, int(D is not None))
    ofi, ob = O.rasterize(V, F, W, H, D)
    assert np.array_equal(fi.numpy(), ofi)
    assert np.array_equal(b.numpy().view(np.uint32), ob.view(np.uint32))


def test_shims_resolve_and_refuse():
    import custom_rasterizer
    import custom_rasterizer_kernel
    from gs_b200 import custom_rasterizer as CR
    assert custom_rasterizer.rasterize is CR.rasterize and custom_rasterizer.interpolate is CR.interpolate
    assert custom_rasterizer_kernel.rasterize_image is CR.rasterize_image
    pos = torch.zeros(1, 3, 4)
    tri = torch.zeros(1, 3, dtype=torch.int32)
    with pytest.raises(TypeError):
        custom_rasterizer.rasterize(pos, tri, 64)                  # an int resolution cannot be indexed
    with pytest.raises(RuntimeError, match="CUDA"):
        custom_rasterizer.rasterize(pos, tri, (8, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        custom_rasterizer_kernel.rasterize_image(pos[0], tri, torch.zeros(0), 8, 8, 1e-6, 0)
    with pytest.raises(RuntimeError, match="CUDA"):
        custom_rasterizer.interpolate(torch.zeros(1, 3, 2), torch.zeros(8, 8, dtype=torch.int32),
                                      torch.zeros(8, 8, 3), tri)
    for fn in (custom_rasterizer_kernel.build_hierarchy, custom_rasterizer_kernel.build_hierarchy_with_feat,
               custom_rasterizer.LoadObj, custom_rasterizer.LoadObjWithTexture, custom_rasterizer.LoadGlb,
               custom_rasterizer.RotatePrimitives):
        with pytest.raises(NotImplementedError):
            fn()


def test_c_abi_scratch_bytes():
    from gs_b200 import _lib
    assert _lib.lib.dr_b200_cr_scratch_bytes(40000, 4096, 4096) == 4096 * 4096 * 8 + 256 + 40000 * 8
    assert _lib.lib.dr_b200_cr_scratch_bytes(1, 0, 8) == 0
