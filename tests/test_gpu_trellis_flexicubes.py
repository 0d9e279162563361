"""TRELLIS FlexiCubes on the H100 (csrc/ngp_flexicubes.cu's attribute passes via gs_b200.isosurface.TrellisFlexiCubes):
every fixture variant of the reference (tests/golden/ref_trellis_flexicubes.npz) and the float64 torch oracle
(oracle/fc_oracle.py, with the colours of test_trellis_flexicubes_cpu.flexicubes_colours) in faces (exactly),
vertices, L_dev, colours and the gradients to x, s, the weights and the raw colours; the no-colour call against
FlexiCubes bit for bit; SparseFeatures2Mesh's layout at res 256 and 128 against the float64 oracle; run-to-run bit
identity; the current stream; host reads; strided views; error paths and empty surfaces."""
import os
import sys
import warnings

import pytest
import torch

from conftest import ROOT
from test_trellis_flexicubes_cpu import (Z, CASES, assert_matches_fixture, case_inputs, flexicubes_colours, oracle_fn,
                                         run_with_grads, variants)

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_flexicubes import trellis_inputs  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _tfc():
    from gs_b200.isosurface import TrellisFlexiCubes
    return TrellisFlexiCubes(device=DEV)


def _cubes(res):
    from gs_b200.isosurface import voxel_grid
    return voxel_grid(res, DEV)[1]


def _cuda_fn(fc, res, training, ws):
    cubes = _cubes(res)

    def fn(x, s, b, a, g, c):
        v, f, L, vc = fc(voxelgrid_vertices=x, scalar_field=s, cube_idx=cubes, resolution=res, weight_scale=ws,
                         beta=b, alpha=a, gamma_f=g, voxelgrid_colors=c, training=training)
        return v, f, L, vc, None
    return fn


def _close(a, b, atol, what):
    err = float((a.double() - b.double()).abs().max()) if a.numel() else 0.0
    assert err <= atol, (what, err)


def _run_both(res, x, s, w, c, given, colours, training, ws, grtol=1e-4):
    """CUDA and the fp64 oracle on the same inputs: the outputs come in the same order, so faces compare exactly."""
    v, f, L, vc, _, g = run_with_grads(_cuda_fn(_tfc(), res, training, ws), x, s, w, c, given, colours, Z)
    ov, of, oL, ovc, keys, og = run_with_grads(oracle_fn(res, training, ws), x, s, w, c, given, colours, Z)
    assert v.dtype == torch.float32 and f.dtype == torch.int64 and L.dtype == torch.float32
    assert v.device == DEV and f.device == DEV and L.device == DEV
    assert v.shape == ov.shape and f.shape == of.shape and L.shape == oL.shape
    assert torch.equal(f, of)
    _close(v, ov, 1e-5, "verts")
    _close(L, oL, 1e-5, "L_dev")
    assert (vc is None) == (not colours)
    if colours:
        assert vc.dtype == torch.float32 and vc.shape == ovc.shape
        _close(vc, ovc, 1e-5, "colours")
    if og is not None:
        for k in ("gx", "gs", "gw", "gc"):
            assert (g[k] is None) == (og[k] is None), k
            if og[k] is not None:
                scale = float(og[k].abs().max())
                err = float((g[k].double() - og[k].double()).abs().max())
                assert err <= grtol * max(scale, 1e-12), (k, err, scale)
    return v, f, L, vc, keys, g


@pytest.mark.parametrize("name", CASES)
def test_fixture_cases_match_the_reference_and_the_oracle(name):
    res, x, s, w, c = case_inputs(Z, name, DEV)
    for ws, given, colours, training in variants(name):
        tag = f"{name}/{ws}/{given}/{colours}/{training}"
        v, f, L, vc, keys, g = _run_both(res, x, s, w, c, given, colours, bool(training), ws)
        assert_matches_fixture(Z, tag, v, f, L, vc, keys, g)


def _bits(t):
    return t.detach().contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _random_inputs(res, seed, C=6):
    from gs_b200.isosurface import voxel_grid
    x, _ = voxel_grid(res, DEV)
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = x * 2 + (1 / res) * torch.tanh(torch.randn(x.shape, generator=gen, device=DEV))
    s = torch.rand(x.shape[0], generator=gen, device=DEV) - 0.1
    w = 0.5 * torch.randn((res ** 3, 21), generator=gen, device=DEV)
    c = torch.randn((x.shape[0], C), generator=gen, device=DEV)
    return x, s, w, c


def _grads_of(fn, x, s, w, c, colour_loss=True):
    x, s, w = (t.detach().clone().requires_grad_(True) for t in (x, s, w))
    c = None if c is None else c.detach().clone().requires_grad_(True)
    v, f, L, vc = fn(x, s, w, c)
    loss = (torch.sin(v @ torch.tensor([0.7, -1.3, 0.4]).to(v))).sum() + v.square().sum() + L.mean()
    if vc is not None and colour_loss:
        loss = loss + (torch.sin(2 * vc) * torch.linspace(-1, 1, vc.shape[1]).to(vc)).sum()
    loss.backward()
    return [v, f, L] + ([vc] if vc is not None else []), [x.grad, s.grad, w.grad] + ([c.grad] if c is not None else [])


@pytest.mark.parametrize("training", [False, True])
def test_without_colours_is_flexicubes_bit_for_bit(training):
    from gs_b200.isosurface import FlexiCubes
    res = 64
    x, s, w, c = _random_inputs(res, seed=21)
    cubes = _cubes(res)
    fc, tfc = FlexiCubes(device=DEV), _tfc()
    node = lambda x_, s_, w_, c_: tuple(fc(x_, s_, cubes, res, beta_fx12=w_[:, :12], alpha_fx8=w_[:, 12:20],
                                           gamma_f=w_[:, 20], training=training)) + (None,)
    trel = lambda x_, s_, w_, c_: tfc(x_, s_, cubes, res, beta=w_[:, :12], alpha=w_[:, 12:20], gamma_f=w_[:, 20],
                                      voxelgrid_colors=c_, training=training)
    out_n, g_n = _grads_of(node, x, s, w, None)
    out_t, g_t = _grads_of(trel, x, s, w, None)
    assert len(out_t) == 3
    for a, b in zip(out_n + g_n, out_t + g_t):
        assert torch.equal(_bits(a), _bits(b))
    # with colours: the same geometry, and the same grad_x when the loss does not involve the colours
    out_c, g_c = _grads_of(trel, x, s, w, c, colour_loss=False)
    for a, b in zip(out_n, out_c[:3]):
        assert torch.equal(_bits(a), _bits(b))
    assert torch.equal(_bits(g_n[0]), _bits(g_c[0]))
    assert out_c[3].shape == (out_c[0].shape[0], 6) and not g_c[3].any()


def _trellis_call(fc, res, cubes, training):
    return lambda x, s, w, c: fc(voxelgrid_vertices=x, scalar_field=s, cube_idx=cubes, resolution=res,
                                 beta=w[:, :12], alpha=w[:, 12:20], gamma_f=w[:, 20], voxelgrid_colors=c,
                                 training=training)


def test_trellis_layout_res256_forward_matches_the_oracle():
    res = 256
    x, s, c, w, cubes = trellis_inputs(res, seed=3, device=DEV)
    with torch.no_grad():
        v, f, L, vc = _trellis_call(_tfc(), res, cubes, False)(x, s, w, c)
        ov, of, oL, _, ovc = flexicubes_colours(x, s, res, w[:, :12], w[:, 12:20], w[:, 20], training=False,
                                                weight_scale=0.99, dtype=torch.float64, attrs=c)
    assert v.shape[0] > 100_000 and vc.shape == (v.shape[0], 6)
    assert torch.equal(f, of)
    _close(v, ov, 1e-5, "verts")
    _close(L, oL, 1e-5, "L_dev")
    _close(vc, ovc, 1e-5, "colours")


@pytest.mark.parametrize("training", [False, True])
def test_trellis_layout_res128_forward_backward_matches_the_oracle(training):
    res = 128
    x, s, c, w, cubes = trellis_inputs(res, seed=4, device=DEV)
    cuda = _trellis_call(_tfc(), res, cubes, training)

    def orc(x_, s_, w_, c_):
        out = flexicubes_colours(x_, s_, res, w_[:, :12], w_[:, 12:20], w_[:, 20], training=training,
                                 weight_scale=0.99, dtype=torch.float64, attrs=c_)
        return out[0], out[1], out[2], out[4]
    (v, f, L, vc), g = _grads_of(cuda, x, s, w, c)
    (ov, of, oL, ovc), og = _grads_of(orc, x, s, w, c)
    assert torch.equal(f, of) and v.shape[0] > 20_000
    for a, b, n in ((v, ov, "verts"), (L, oL, "L_dev"), (vc, ovc, "colours")):
        _close(a.detach(), b.detach(), 1e-5, n)
    for a, b, n in zip(g, og, ("x", "s", "w", "c")):
        scale = float(b.abs().max())
        err = float((a.double() - b.double()).abs().max())
        assert scale > 0 and err <= 1e-4 * scale, (n, err, scale)


def test_two_runs_are_bit_identical_with_colours():
    res = 96
    x, s, w, c = _random_inputs(res, seed=22)
    fn = _trellis_call(_tfc(), res, _cubes(res), True)
    a = _grads_of(fn, x, s, w, c)
    b = _grads_of(fn, x, s, w, c)
    for p, q in zip(a[0] + a[1], b[0] + b[1]):
        assert torch.equal(_bits(p), _bits(q))


def test_runs_on_the_current_stream():
    res = 48
    x, s, w, c = _random_inputs(res, seed=23)
    fn = _trellis_call(_tfc(), res, _cubes(res), True)
    ref = _grads_of(fn, x, s, w, c)
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)              # keeps the side stream busy: work on another stream would race
        got = _grads_of(fn, x, s, w, c)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for p, q in zip(ref[0] + ref[1], got[0] + got[1]):
        assert torch.equal(_bits(p), _bits(q))


def test_one_host_read_per_forward_and_none_in_the_backward():
    from gs_b200 import _lib
    res = 64
    x, s, w, c = _random_inputs(res, seed=24)
    s, w, c = (t.clone().requires_grad_(True) for t in (s, w, c))
    fn = _trellis_call(_tfc(), res, _cubes(res), True)
    fn(x, s, w, c)                                 # recognises cube_idx (a one-time check)
    torch.cuda.synchronize()
    n0 = _lib.lib.gs_b200_launch_count()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            v, f, L, vc = fn(x, s, w, c)
        n1 = _lib.lib.gs_b200_launch_count()
        loss = v.square().sum() + L.mean() + vc.square().sum()
        torch.cuda.set_sync_debug_mode("error")
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    n2 = _lib.lib.gs_b200_launch_count()
    syncs = [r for r in rec if "synchroniz" in str(r.message)]
    assert len(syncs) == 1, [str(r.message) for r in syncs]
    assert n2 - n1 == 3                            # quad partials, per-cube gradients, per-point gather
    assert n1 - n0 >= 3
    assert c.grad is not None and c.grad.any()


@pytest.mark.parametrize("training", [False, True])
def test_strided_views_match_contiguous_copies(training):
    res = 40
    x, s, w, c = _random_inputs(res, seed=25)
    fn = _trellis_call(_tfc(), res, _cubes(res), training)
    # SparseFeatures2Mesh's views: sdf and colours are columns of one [P,10] array, the weights columns of [F,21]
    dense = torch.cat([s[:, None], torch.zeros_like(x), c], 1).requires_grad_(True)
    wd = w.clone().requires_grad_(True)
    v2, f2, L2, vc2 = fn(x, dense[:, 0], wd, dense[:, 4:])
    loss = v2.square().sum() + L2.mean() + vc2.square().sum()
    loss.backward()
    assert dense[:, 4:].stride() == (10, 1)
    ref = [t.detach().clone().requires_grad_(True) for t in (s, w, c)]
    v3, f3, L3, vc3 = fn(x, ref[0], ref[1], ref[2])
    (v3.square().sum() + L3.mean() + vc3.square().sum()).backward()
    for a, b in ((v2, v3), (f2, f3), (L2, L3), (vc2, vc3), (dense.grad[:, 0], ref[0].grad), (wd.grad, ref[1].grad),
                 (dense.grad[:, 4:], ref[2].grad)):
        assert torch.equal(_bits(a), _bits(b))
    assert not dense.grad[:, 1:4].any()


def test_error_paths():
    from gs_b200 import _lib
    fc = _tfc()
    res = 8
    x, s, w, c = _random_inputs(res, seed=26, C=3)
    cubes = _cubes(res)
    F = res ** 3
    call = lambda **kw: fc(**{**dict(voxelgrid_vertices=x, scalar_field=s, cube_idx=cubes, resolution=res,
                                     voxelgrid_colors=c), **kw})
    bad = [(dict(voxelgrid_vertices=x[:, :2]), "'voxelgrid_vertices' should be a tensor of shape (num_vertices, 3)"),
           (dict(voxelgrid_vertices=x.tolist()), "'voxelgrid_vertices' should be"),
           (dict(scalar_field=s[:, None]), "'scalar_field' should be a tensor of shape (num_vertices,)"),
           (dict(scalar_field=s[:-1]), "'scalar_field' should be"),
           (dict(cube_idx=cubes[:, :7]), "'cube_idx' should be a tensor of shape (num_cubes, 8)"),
           (dict(beta=w[:-1, :12]), "'beta' should be a tensor of shape (num_cubes, 12)"),
           (dict(alpha=w[:, :7]), "'alpha' should be a tensor of shape (num_cubes, 8)"),
           (dict(gamma_f=w[:, 20:]), "'gamma_f' should be a tensor of shape (num_cubes,)"),
           (dict(voxelgrid_colors=c[:-1]), "'voxelgrid_colors' should be a tensor of shape (num_vertices, C)"),
           (dict(voxelgrid_colors=c[:, :0]), "'voxelgrid_colors' should be"),
           (dict(voxelgrid_colors=c[:, 0]), "'voxelgrid_colors' should be")]
    for kw, msg in bad:
        with pytest.raises(AssertionError, match=msg.replace("(", r"\(").replace(")", r"\)")):
            call(**kw)
    with pytest.raises(TypeError):
        call(voxelgrid_vertices=x.cpu(), scalar_field=s.cpu(), cube_idx=cubes.cpu(), voxelgrid_colors=c.cpu())
    with pytest.raises(TypeError):
        call(voxelgrid_colors=c.cpu())
    with pytest.raises(ValueError):
        call(cube_idx=cubes.flip(0).contiguous())
    v, f, L, vc = call(beta=w[:, :12], alpha=w[:, 12:20], gamma_f=w[:, 20], qef_reg_scale=0.5)
    assert v.shape[0] > 0 and vc.shape == (v.shape[0], 3)
    # the C ABI checks the attribute arguments and reports through last_error
    host = (__import__("ctypes").c_ulonglong * 4)(1, 1, 0, 1)
    P = lambda t: __import__("ctypes").c_void_p(t.data_ptr())
    out = torch.empty(16, device=DEV)
    for attrs, stride, C, msg in ((None, 3, 3, "NULL attributes"), (P(c), 3, 0, "C >= 1"), (P(c), 2, 3, "C >= 1")):
        rc = _lib.lib.ngp_b200_flexicubes_write_attrs(P(x), P(s), None, 0, None, 0, None, 0, res, res, res, 0.99, 0,
                                                      host, P(out), P(out), P(out), attrs, stride, C, P(out), P(out),
                                                      None)
        assert rc == 1 and msg in _lib.last_error() and "flexicubes_write_attrs" in _lib.last_error()
    assert _lib.lib.ngp_b200_flexicubes_backward_attrs_workspace_bytes(host, 1, 0) == 0


@pytest.mark.parametrize("training", [False, True])
def test_empty_surface_returns_the_reference_shapes(training):
    from gs_b200.isosurface import voxel_grid
    fc = _tfc()
    x, cubes = voxel_grid(6, DEV)
    for sv in (1.0, -1.0):
        for C in (None, 6):
            s = torch.full((x.shape[0],), sv, device=DEV, requires_grad=True)
            c = None if C is None else torch.randn((x.shape[0], C), device=DEV, requires_grad=True)
            v, f, L, vc = fc(x, s, cubes, 6, voxelgrid_colors=c, training=training)
            assert v.shape == (0, 3) and f.shape == (0, 3) and L.shape == (0,) and f.dtype == torch.int64
            if C is None:
                assert vc is None
                (v.sum() + L.sum()).backward()
            else:
                assert vc.shape == (0, C) and vc.dtype == torch.float32
                (v.sum() + L.sum() + vc.sum()).backward()
                assert c.grad is not None and not c.grad.any()
            assert s.grad is not None and not s.grad.any()
