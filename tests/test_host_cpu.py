"""CPU tests of the host side (no GPU): the C-ABI library loads and exports every symbol the header declares,
struct layouts agree with the header, the reference-facing Python interface validates like the package does,
and the host camera logic matches the oracle / reference fixtures."""
import ctypes
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

HEADER = os.path.join(ROOT, "include", "gs_b200.h")


def _ensure_built():
    lib = os.path.join(ROOT, "comfyui-3d-pack_b200", "gs_b200", "libgs_b200.so")
    if not os.path.exists(lib):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    return lib


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(_ensure_built())
    src = open(HEADER).read()
    names = set(re.findall(r"\b(gs_b200_[a-z0-9_]+)\s*\(", src))
    names -= {"gs_b200_alloc_fn"}
    assert len(names) >= 14
    for n in sorted(names):
        assert hasattr(lib, n), f"{n} declared in include/gs_b200.h but not exported"
    lib.gs_b200_abi_version.restype = ctypes.c_int32
    assert lib.gs_b200_abi_version() == 1


def test_all_five_headers_are_plain_c_and_every_declared_entry_point_is_exported():
    """include/*.h (gs, dr, ngp, attention, points): each compiles as C on its own (no C++ / torch types in the
    boundary) and every function it declares is an exported symbol of libgs_b200.so."""
    lib = ctypes.CDLL(_ensure_built())
    inc = os.path.join(ROOT, "include")
    headers = sorted(f for f in os.listdir(inc) if f.endswith(".h"))
    assert headers == ["dr_b200.h", "gs_b200.h", "gs_b200_attn.h", "gs_b200_pts.h", "ngp_b200.h"]
    total = 0
    for h in headers:
        subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-x", "c", os.path.join(inc, h)], check=True)
        src = re.sub(r"/\*.*?\*/", "", open(os.path.join(inc, h)).read(), flags=re.S)
        prefix = h.split("_")[0]
        names = set(re.findall(r"\b(%s_b200_[a-z0-9_]+)\s*\(" % prefix, src))
        names -= {"gs_b200_alloc_fn"}
        assert names, h
        for n in sorted(names):
            assert hasattr(lib, n), f"{n} declared in include/{h} but not exported"
        total += len(names)
    assert total >= 45


def test_ctypes_structs_match_header_layout():
    from gs_b200 import _lib
    code = r'''
    #include <stdio.h>
    #include <stddef.h>
    #include "gs_b200.h"
    int main(void){ printf("%zu %zu %zu %zu %zu %zu\n", sizeof(gs_b200_view), offsetof(gs_b200_view, campos),
        sizeof(gs_b200_state), offsetof(gs_b200_state, num_rendered), offsetof(gs_b200_state, owned), offsetof(gs_b200_view, viewmatrix)); return 0; }
    '''
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c"); exe = os.path.join(d, "t")
        open(c, "w").write(code)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    sv, oc, ss, onr, oo, ovm = map(int, out)
    assert ctypes.sizeof(_lib.View) == sv and _lib.View.campos.offset == oc and _lib.View.viewmatrix.offset == ovm
    assert ctypes.sizeof(_lib.State) == ss and _lib.State.num_rendered.offset == onr and _lib.State.owned.offset == oo


def test_ctypes_binding_is_derived_from_every_header_in_include():
    """gs_b200._lib binds every function include/*.h declares, with one argtype per declared parameter; a few
    signatures are pinned by hand (every row of the C -> ctypes mapping), the header constants reach Python, and a
    by-value type the mapping does not know is refused rather than guessed."""
    from gs_b200 import _lib
    declared = {}
    for h in sorted(f for f in os.listdir(os.path.join(ROOT, "include")) if f.endswith(".h")):
        src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", h)).read(), flags=re.S)
        for name, params in re.findall(r"\b((?:gs|dr|ngp)_b200_\w+)\s*\(([^()]*)\)\s*;", src):
            declared[name] = 0 if params.strip() == "void" else params.count(",") + 1
    bound = {n for n, f in vars(_lib.lib).items() if isinstance(f, _lib.lib._FuncPtr)}
    assert len(declared) == 106 and bound == set(declared)
    assert len(_lib.lib.gs_b200_debug_preprocess_views.argtypes) == 17
    for name, nparams in declared.items():
        assert len(getattr(_lib.lib, name).argtypes) == nparams, name

    I, L, F, D, P, S = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_double, ctypes.c_void_p, ctypes.c_size_t
    expected = {
        "ngp_b200_grid_encode_fwd": (I, (P, L, P, P, I, F, D, I, P, P)),
        "gs_b200_adam_step": (I, (I, I, P, D, D, F, I, F, P, P, P, P, P)),
        "gs_b200_sort_scratch_bytes": (S, (L,)),
        "gs_b200_launch_count": (L, ()),
        "gs_b200_last_error": (ctypes.c_char_p, ()),
        "gs_b200_profile_enable": (None, (I,)),
        "gs_b200_rasterize_forward": (I, (ctypes.POINTER(_lib.View), I, I) + (P,) * 11 +
                                      (_lib.ALLOC_FN, P, ctypes.POINTER(_lib.State), P)),
        "gs_b200_step_device_hook": (I, (I, I, I, I, F, P, P, I, I) + (P,) * 9 + (_lib.VIEW_HOOK, P, P, P)),
        "gs_b200_set_grad_sink": (I, (_lib.GRAD_SINK, P, I)),
        "gs_b200_attn_forward": (I, (I, I, I, I) + (P, L, L) * 3 + (P, P, L, L, L, L, F, P, P)),
        "gs_b200_pts_rasterize": (I, (I, L, I, I, I, F, I) + (P,) * 11),
    }
    for name, (restype, argtypes) in expected.items():
        fn = getattr(_lib.lib, name)
        assert (fn.restype, tuple(fn.argtypes)) == (restype, argtypes), name

    assert _lib.SPCONV_MAX_ROWS == (1 << 30) - 1 and _lib.PN2_FPS_ONCHIP_MAX == 16384
    assert _lib.SCATTER_MAX_DIMS == 8 and _lib.BUF_SCRATCH == 3
    assert _lib.NSTAGES == len(_lib.STAGE_NAMES) == 9

    assert _lib.prototypes("int32_t gs_b200_x(const uint8_t* x, void* stream);") == {"gs_b200_x": (I, [P, P])}
    with pytest.raises(ImportError, match="gs_b200_x.*uint8_t"):
        _lib.prototypes("int32_t gs_b200_x(uint8_t x);")


def test_dr_and_ngp_entry_points_refuse_bad_arguments_with_their_messages():
    """Every dr_b200_* / ngp_b200_* entry point, called with arguments that fail its first check, returns 1 and sets
    gs_b200_last_error() to exactly "<entry point>: <message>", with no GPU work.  The size and capability queries,
    which have no error path, return their documented values (0 for invalid arguments)."""
    from gs_b200 import _lib
    lib, N = _lib.lib, None
    refused = {
        "dr_b200_rasterize_fwd": ((N, N, -1, 0, 0, 1, 1, N, N, N, N), "bad sizes"),
        "dr_b200_rasterize_bwd": ((N, N, 1, 1, 1, 1, 1, N, N, N, N), "NULL pointer"),
        "dr_b200_interpolate_fwd": ((N, 1, N, N, N, 1, 1, 1, 1, 1, 1, N, N, N), "NULL pointer"),
        "dr_b200_interpolate_bwd": ((N, 1, N, N, N, 1, 1, 1, 1, 1, 1, N, N, N, N, N, N), "NULL pointer"),
        "dr_b200_texture_fwd": ((N, 1, 1, 1, 1, N, 1, 1, 1, 0, N, N), "bad argument"),
        "dr_b200_texture_bwd": ((N, 1, 1, 1, 1, N, 1, 1, 1, 0, N, N, N, N), "NULL pointer"),
        "dr_b200_edge_opposites": ((N, 1, 3, N, N, N), "NULL pointer"),
        "dr_b200_antialias_fwd": ((N, N, N, N, N, 1, 1, 1, 1, 1, 1, N, N), "NULL pointer"),
        "dr_b200_antialias_bwd": ((N, N, N, N, N, 1, 1, 1, 1, 1, 1, N, N, N, N), "NULL pointer"),
        "dr_b200_cr_rasterize": ((N, -1, N, 0, N, 1, 1, 0.0, N, N, N, N), "bad sizes"),
        "dr_b200_cr_interpolate_fwd": ((N, -1, 1, N, 0, N, N, 0, 0, 0, N, N), "bad sizes"),
        "dr_b200_cr_interpolate_bwd": ((N, -1, 1, N, 0, N, N, 0, 0, 0, N, N, N, N, N), "bad sizes"),
        "dr_b200_uvbake_rasterize": ((N, 0, N, 0, N, 0, 0, 0, N, N), "bad sizes"),
        "dr_b200_uvbake_interpolate": ((N, 0, N, 0, N, N, 0, 0, 0, N), "bad sizes"),
        "ngp_b200_grid_encode_fwd": ((N, 1, N, N, 1, 1.0, 2.0, 16, N, N), "NULL pointer"),
        "ngp_b200_grid_encode_bwd": ((N, 1, N, 1, 1.0, 2.0, 16, N, N, N), "NULL pointer"),
        "ngp_b200_grid_tv_grad": ((N, 1, N, N, 1, 1.0, 2.0, 16, 1.0, N, N), "NULL pointer"),
        "ngp_b200_march_count": ((N, N, 1, N, 1, N, 0.0, 1.0, 0.1, N, N, N, N, N, N), "NULL pointer"),
        "ngp_b200_march_write": ((N, N, 1, 1, N, 0.0, 1.0, 0.1, N, N, N, N, N, N, N), "NULL pointer"),
        "ngp_b200_ray_ranges": ((N, 1, 1, N, N), "NULL pointer"),
        "ngp_b200_weights_fwd": ((N, N, N, N, 1, N, N, N, N), "NULL ranges"),
        "ngp_b200_weights_bwd": ((N, N, N, N, 1, N, N, N, N, N, N, N), "NULL ranges"),
        "ngp_b200_accumulate_fwd": ((N, N, 1, N, 1, N, N), "NULL pointer"),
        "ngp_b200_accumulate_bwd": ((N, N, 1, N, 1, N, N, N, N), "NULL pointer"),
        "ngp_b200_mlp2_fwd": ((N, 1, 24, 32, 1, N, N, N, N), "NULL pointer"),
        "ngp_b200_mlp2_bwd": ((N, 1, 24, 32, 1, N, N, N, N, N, N, N), "NULL pointer"),
    }
    for name, (args, msg) in refused.items():
        assert getattr(lib, name)(*args) == 1, name
        assert _lib.last_error() == f"{name}: {msg}"

    assert lib.dr_b200_rasterize_scratch_bytes(1, 1, 1, 1) == 8 + 256 + (2 + 4096) * 8 + 4
    assert lib.dr_b200_topology_scratch_bytes(1) == 4 * 256 + lib.gs_b200_sort_scratch_bytes(3) + 256
    assert lib.dr_b200_cr_scratch_bytes(-1, 1, 1) == 0 and lib.dr_b200_cr_scratch_bytes(1, 2, 2) == 2 * 2 * 8 + 256 + 8
    assert lib.dr_b200_uvbake_scratch_bytes(1, 1 << 16) == 0 and lib.dr_b200_uvbake_scratch_bytes(1, 2) == 256 + 16 + 8
    assert lib.ngp_b200_march_scratch_bytes(1, 64) - lib.ngp_b200_march_scratch_bytes(1, 32) == (64 ** 3 - 32 ** 3) // 8
    assert lib.ngp_b200_mlp2_supported(24, 32, 1) == 1 and lib.ngp_b200_mlp2_supported(16, 32, 1) == 0


def test_rasterizer_entry_points_refuse_bad_arguments_with_their_messages():
    """Every argument-taking gs_b200_* entry point of the rasterizer and the multi-view step, called with arguments
    that fail its first check, returns 1 (gs_b200_step_view_chunks: -1) and sets gs_b200_last_error() to exactly
    "<entry point>: <message>", before any CUDA call: without a GPU, one would set a CUDA error instead."""
    from gs_b200 import _lib
    lib = _lib.lib

    def call(name, *lead):               # the given leading arguments, then zero / NULL for all the others
        fn = getattr(lib, name)
        return fn(*lead, *(t() for t in fn.argtypes[len(lead):]))

    sink = _lib.GRAD_SINK(lambda user, first, count, stream: None)
    refused = {      # name: (leading arguments, message); V = 0 fails every step entry first
        "gs_b200_set_tile_culling": ((3,), "tile culling mode must be 0, 1 or 2"),
        "gs_b200_rasterize_forward": ((), "NULL view field"),
        "gs_b200_rasterize_backward": ((), "NULL view field"),
        "gs_b200_debug_sorted_keys": ((), "NULL argument"),
        "gs_b200_debug_preprocess_backward": ((), "NULL view field"),
        "gs_b200_debug_preprocess_backward_multi": ((), "bad argument"),
        "gs_b200_set_grad_sink": ((sink,), "nchunks must be 1..64"),
        "gs_b200_step_device": ((), "bad argument"),
        "gs_b200_step_device_hook": ((), "bad argument"),
        "gs_b200_image_loss": ((), "NULL argument"),
        "gs_b200_step_device_train": ((), "bad argument"),
        "gs_b200_render_views": ((), "bad argument"),
        "gs_b200_debug_sort_segmented": ((), "bad argument"),
        "gs_b200_debug_bin_views": ((), "bad argument"),
        "gs_b200_debug_preprocess_views": ((), "bad argument"),
        "gs_b200_step_host": ((), "bad argument"),
        "gs_b200_step_host_dev_grads": ((), "bad argument"),
    }
    for name, (lead, msg) in refused.items():
        assert call(name, *lead) == 1, name
        assert _lib.last_error() == f"{name}: {msg}"
    assert call("gs_b200_step_view_chunks") == -1
    assert _lib.last_error() == "gs_b200_step_view_chunks: bad argument"


def test_settings_namedtuple_field_order_matches_reference_call_site():
    # main_3DGS_renderer.py:849-862 constructs it by keyword; LGM/TRELLIS too. Order = the package's NamedTuple.
    from diff_gaussian_rasterization import GaussianRasterizationSettings
    assert GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix",
        "sh_degree", "campos", "prefiltered", "debug")


def test_rasterizer_argument_validation_matches_package_messages():
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    z = torch.zeros
    rs = GaussianRasterizationSettings(16, 16, 1.0, 1.0, z(3), 1.0, torch.eye(4), torch.eye(4), 0, z(3), False, False)
    r = GaussianRasterizer(raster_settings=rs)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), scales=z(1, 3), rotations=z(1, 4))
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), shs=z(1, 1, 3), colors_precomp=z(1, 3), scales=z(1, 3), rotations=z(1, 4))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), colors_precomp=z(1, 3))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), colors_precomp=z(1, 3), scales=z(1, 3), rotations=z(1, 4), cov3D_precomp=z(1, 6))


def test_no_cpu_fallback_cpu_tensors_are_rejected():
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    z = torch.zeros
    rs = GaussianRasterizationSettings(16, 16, 1.0, 1.0, z(3), 1.0, torch.eye(4), torch.eye(4), 0, z(3), False, False)
    with pytest.raises(RuntimeError, match="no CPU path"):
        GaussianRasterizer(rs)(means3D=z(1, 3), means2D=z(1, 3), opacities=z(1, 1), colors_precomp=z(1, 3), scales=z(1, 3), rotations=z(1, 4))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "comfyui-3d-pack_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from\s+oracle|import\s+oracle|from\s+\.*gs_oracle|import\s+gs_oracle)", txt, flags=re.M), f


def test_host_camera_matches_reference_fixtures_and_oracle():
    from gs_b200 import camera
    from oracle import gs_oracle as O
    g = np.load(os.path.join(GOLDEN, "ref_camera.npz"))
    for i in range(3):
        W, H, fovy = g[f"dims{i}"]
        fy = np.deg2rad(fovy); fx = 2 * np.arctan(np.tan(fy / 2) * W / H)
        mc = camera.MiniCam(g[f"c2w{i}"], int(W), int(H), fy, fx, 0.01, 100.0, device="cpu")
        assert np.allclose(mc.world_view_transform.numpy(), g[f"wvt{i}"], atol=1e-6)
        assert np.allclose(mc.full_proj_transform.numpy(), g[f"full{i}"], atol=1e-5)
        assert np.allclose(mc.camera_center.numpy(), g[f"center{i}"], atol=1e-7)
    for el, az in [(0, 0), (30, 100), (-40, -170)]:
        assert np.allclose(camera.orbit_camera(el, az, 1.75), O.orbit_camera(el, az, 1.75), atol=1e-6)
    v = camera.orbit_views(8, 1920, 1080)
    st = O.minicam_settings(O.orbit_camera(0, 45.0, 1.75), 1920, 1080, 49.1)
    assert np.allclose(v[1, :16], st.viewmatrix.reshape(-1).numpy(), atol=1e-6)
    assert np.allclose(v[1, 16:32], st.projmatrix.reshape(-1).numpy(), atol=1e-5)
    assert abs(v[1, 38] - st.tanfovx) < 1e-6 and abs(v[1, 39] - st.tanfovy) < 1e-6


def test_gs_ply_wire_format_roundtrip_and_property_order(tmp_path):
    from gs_b200 import ply
    g = torch.Generator().manual_seed(0)
    N, M = 37, 16
    d = dict(xyz=torch.randn(N, 3, generator=g), shs=torch.randn(N, M, 3, generator=g), opacity=torch.randn(N, 1, generator=g),
             scaling=torch.randn(N, 3, generator=g), rotation=torch.randn(N, 4, generator=g))
    path = str(tmp_path / "g.ply")
    ply.write_gs_ply(path, **d)
    head = open(path, "rb").read(4096).split(b"end_header\n")[0].decode().splitlines()
    props = [l.split()[-1] for l in head if l.startswith("property")]
    # mesh_utils.py:333-344 (construct_list_of_gs_attributes) order
    assert props[:9] == ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"]
    assert props[9] == "f_rest_0" and props[9 + 44] == "f_rest_44" and props[-8:] == ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    assert all(l.startswith("property float ") for l in head if l.startswith("property"))
    back = ply.read_gs_ply(path)
    for k in d:
        assert torch.equal(back[k], d[k]), k
    # channel-major SH planes, as to_ply's transpose(1,2).flatten (main_3DGS_renderer.py:475-484)
    rows = ply.pack_rows(**d)
    assert float(rows[5, 9 + 1 * 15 + 3]) == float(d["shs"][5, 4, 1])          # f_rest_{c*(M-1)+k} = coeff k+1 of channel c
    assert ply.max_sh_degree_from_properties(45) == 3 and ply.max_sh_degree_from_properties(0) == 0


def test_switch_axis_and_scale_matches_the_reference_sequence():
    """gs_b200.ply.switch_axis_and_scale against a step-by-step restatement of switch_ply_axis_and_scale
    (mesh_processer/mesh_utils.py:446-472) in numpy, including the in-place column permutation of switch_vector_axis
    (:433-443) and the odd-inversion sign flip; quaternion <-> axis-angle round trip is the identity on unit quaternions."""
    import numpy as np
    import torch
    from gs_b200 import ply
    rng = np.random.RandomState(0)
    n = 257
    q = rng.normal(size=(n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[0] = [1, 0, 0, 0]; q[1] = [-1, 0, 0, 0]                       # zero vector part: the k = 2 / k = 0.5 branches
    f = dict(xyz=torch.from_numpy(rng.normal(size=(n, 3)).astype(np.float32)), shs=torch.zeros(n, 4, 3), opacity=torch.zeros(n, 1),
             scaling=torch.from_numpy(rng.normal(size=(n, 3)).astype(np.float32)), rotation=torch.from_numpy(q.astype(np.float32)))
    rt = ply.axis_angle_to_quaternion(ply.quaternion_to_axis_angle(f["rotation"]))
    same = torch.minimum((rt - f["rotation"]).abs().amax(1), (rt + f["rotation"]).abs().amax(1))     # q and -q are one rotation
    assert float(same.max()) < 1e-5
    for axis, scale, inv in (([2, 0, 1], [1.0, -1.0, 1.0], 1), ([0, 2, 1], [2.0, 2.0, 2.0], 0), ([0, 1, 2], [1.0, 1.0, 1.0], 2)):
        out = ply.switch_axis_and_scale(f, axis, scale, inv)
        sc = np.asarray(scale, dtype=np.float32)
        xyz = (f["xyz"].numpy() * sc)[:, axis]
        w, v = q[:, 0], q[:, 1:]
        s = np.linalg.norm(v, axis=1)
        two_theta = 2 * np.where(w < 0, np.arctan2(-s, -w), np.arctan2(s, w))
        k = np.where(s > 0, two_theta / np.where(s > 0, s, 1), 2.0)
        aa = ((v * k[:, None]) * sc)[:, axis]
        if inv % 2:
            aa = -aa
        t = np.linalg.norm(aa, axis=1)
        kk = np.where(t > 0, np.sin(0.5 * t) / np.where(t > 0, t, 1), 0.5)
        ref_q = np.concatenate([np.where(t > 0, np.cos(0.5 * t), 1.0)[:, None], aa * kk[:, None]], 1)
        assert np.allclose(out["xyz"].numpy(), xyz, atol=1e-6)
        assert np.array_equal(out["scaling"].numpy(), f["scaling"].numpy()[:, axis])
        assert np.allclose(out["rotation"].numpy(), ref_q, atol=2e-6)
        assert out["shs"] is f["shs"] and out["opacity"] is f["opacity"]


def test_bench_harness_imports_without_a_gpu_and_the_clock_poller_degrades_gracefully():
    """bench.py must be importable on the CPU box (the driver parses its line there), `--impl reference` and the three
    workloads must be selectable, and the nvidia-smi poller must neither raise nor report clocks when the tool is absent
    or prints nothing (clocks = None is what the line then carries, never a made-up figure)."""
    import importlib
    import shutil
    import sys
    sys.path.insert(0, ROOT)
    bench = importlib.import_module("bench")
    for interval in (20, 100):
        c = bench.Clocks(0, interval)
        out = c.stop()
        assert set(out) >= {"sm_mhz", "sm_max_mhz", "reasons"}
        if shutil.which("nvidia-smi") is None:
            assert c.p is None and out["sm_mhz"] is None and out["reasons"] == []
    src = open(bench.__file__).read()
    for token in ("--impl", "--workload", "--gpus", "--steps", "--warmup", '"roofline"', '"cpu_baseline"', '"e2e"', '"gpu_launches"', '"clocks"'):
        assert token in src, token
