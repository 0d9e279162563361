"""TRELLIS FlexiCubes (vertex colours) without a GPU: the torch oracle (oracle/fc_oracle.py for the geometry,
`flexicubes_colours` here for the colours) in fp64 and fp32 against the reference's own outputs and gradients
(tests/golden/ref_trellis_flexicubes.npz, written by tests/golden/make_golden_trellis_flexicubes.py), colours and
colour gradients included, and the closed-form grid against the digests of the reference's construct_dense_grid.
The fixture helpers here are shared with tests/test_gpu_trellis_flexicubes.py and scripts/bench_flexicubes.py."""
import hashlib
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import fc_oracle as O

Z = np.load(os.path.join(GOLDEN, "ref_trellis_flexicubes.npz"))
CASES = ["trellis", "random", "c1", "inside", "outside"]


def variants(name):
    """(weight_scale, weights given, colours given, training) of every fixture entry of a case."""
    wss = (0.99, 0.5) if name == "random" else (0.99,)
    return [(ws, g, c, t) for ws in wss for g in (1, 0) for c in (1, 0) for t in (0, 1)]


def case_inputs(z, name, device="cpu"):
    """(res, x fp32 [P,3], s fp32 [P], weight fp32 [F,21], raw colours fp32 [P,C]) of a fixture case, exactly."""
    res = tuple(int(r) for r in z[f"{name}/res"])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    if name == "trellis":
        # dense defaults (get_defomed_verts at zero deform, sdf 1, zero colours and weights), then the stored rows
        R = res[0]
        a = torch.arange(R + 1)
        pts = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
        x = pts / R - 0.5 + (1 - 1e-8) / (R * 2) * torch.tanh(torch.zeros(pts.shape))
        prows, wrows = (torch.from_numpy(z[f"trellis/{k}"]).long() for k in ("prows", "wrows"))
        s = torch.ones(x.shape[0])
        c = torch.zeros((x.shape[0], z["trellis/c"].shape[1]))
        w = torch.zeros((R ** 3, 21))
        x[prows], s[prows], c[prows] = t(z["trellis/x"]).cpu(), t(z["trellis/s"]).cpu(), t(z["trellis/c"]).cpu()
        w[wrows] = t(z["trellis/w"]).cpu()
        return res, x.to(device), s.to(device), w.to(device), c.to(device)
    from gs_b200.isosurface import voxel_grid
    grid, _ = voxel_grid(res, device)
    x = grid * 2 + t(z[f"{name}/xq"]).float() / 4096
    return (res, x, t(z[f"{name}/sq"]).float() / 1024, t(z[f"{name}/wq"]).float() / 32,
            t(z[f"{name}/cq"]).float() / 16)


def loss_of(v, L, vc, z):
    fa = torch.tensor(z["functional"], dtype=torch.float64)
    out = O.functional(v, L, fa[:3], fa[3:6], float(fa[6]))
    if vc is not None:
        k = torch.tensor(z["colour_functional"][:vc.shape[1]]).to(vc)
        out = out + (torch.sin(2 * vc) * k).sum()
    return out


def run_with_grads(fn, x, s, w, c, given, colours, z):
    """Runs fn(x, s, beta, alpha, gamma, colours) -> (verts, faces, L, colours or None, keys or None) and
    differentiates the fixture's functional.  Returns (verts, faces, L, colours, keys, {"gx", "gs", "gw", "gc"}),
    gradients None when the mesh is empty."""
    x = x.detach().clone().requires_grad_(True)
    s = s.detach().clone().requires_grad_(True)
    w = w.detach().clone().requires_grad_(True)
    c = c.detach().clone().requires_grad_(True)
    kw = (w[:, :12], w[:, 12:20], w[:, 20]) if given else (None, None, None)
    v, f, L, vc, keys = fn(x, s, *kw, c if colours else None)
    grads = None
    if v.shape[0]:
        loss_of(v, L, vc, z).backward()
        grads = {"gx": x.grad, "gs": s.grad, "gw": w.grad if given else None, "gc": c.grad if colours else None}
    return v.detach(), f, L.detach(), None if vc is None else vc.detach(), keys, grads


def flexicubes_colours(x, s, res, beta=None, alpha=None, gamma=None, training=False, weight_scale=0.99, dtype=None,
                       attrs=None):
    """O.flexicubes with TRELLIS's vertex colours, restated in torch and differentiated by autograd: returns
    (vertices, faces, L_dev, keys) and, when raw attrs [N,C] are given, vertex colours [V,C] as a fifth element.
    sigmoid(attrs) is crossed on each (dual vertex, group edge) entry with the end weights s * alpha of its position
    and averaged with beta; in training each quad centre takes the gamma-weighted diagonal means.  The entries and
    quads are read off the geometry oracle's outputs: an L_dev entry's keys name its dual vertex (cube * 4096 + edge
    mask) and cube edge, in (cube, group, edge) order, and training faces come four per quad, (q_i, q_i+1, centre)."""
    v, f, L, keys = O.flexicubes(x, s, res, beta, alpha, gamma, training=training, weight_scale=weight_scale,
                                 dtype=dtype)
    if attrs is None:
        return v, f, L, keys
    dt = dtype or x.dtype
    dev = x.device
    ws = weight_scale
    vkeys, lvkeys, ledges = keys
    nvd = int((vkeys >= 0).sum())                       # dual vertices first, then (training) centres, keyed < 0
    srt, perm = vkeys[:nvd].sort()
    ent_vd = perm[torch.searchsorted(srt, lvkeys)]
    ent_cube = lvkeys // 4096
    corners, _ = O.grid_ids(res, dev)
    ce = torch.tensor(O.CUBE_EDGES, device=dev).reshape(12, 2)
    ca, cb = ce[ledges, 0], ce[ledges, 1]
    pa, pb = corners[ent_cube, ca], corners[ent_cube, cb]
    s = s.to(dt)
    al = torch.tanh(alpha.to(dt)) * ws + 1 if alpha is not None else None
    be = torch.tanh(beta.to(dt)) * ws + 1 if beta is not None else None
    wa = s[pa] * (al[ent_cube, ca] if al is not None else 1)
    wb = s[pb] * (al[ent_cube, cb] if al is not None else 1)
    c = torch.sigmoid(attrs.to(dt))
    uc = (c[pa] * wb[:, None] - c[pb] * wa[:, None]) / (wb - wa)[:, None]
    b = (be[ent_cube, ledges] if be is not None else torch.ones(ledges.shape, dtype=dt, device=dev))[:, None]
    vc = torch.zeros((nvd, c.shape[1]), dtype=dt, device=dev).index_add(0, ent_vd, uc * b) / \
        torch.zeros((nvd, 1), dtype=dt, device=dev).index_add(0, ent_vd, b)
    if training:
        q = f.reshape(-1, 4, 3)[:, :, 0]
        ga = torch.sigmoid(gamma.to(dt)) * ws + (1 - ws) / 2 if gamma is not None else \
            torch.ones(corners.shape[0], dtype=dt, device=dev)
        g = ga[vkeys[:nvd] // 4096][q]
        g02, g13 = g[:, 0] * g[:, 2], g[:, 1] * g[:, 3]
        w = vc[q]
        vc = torch.cat([vc, (((w[:, 0] + w[:, 2]) / 2) * g02[:, None] + ((w[:, 1] + w[:, 3]) / 2) * g13[:, None]) /
                        (g02 + g13 + 1e-8)[:, None]])
    return v, f, L, keys, vc


def oracle_fn(res, training, ws, dtype=torch.float64):
    def fn(x, s, b, a, g, c):
        out = flexicubes_colours(x, s, res, b, a, g, training=training, weight_scale=ws, dtype=dtype, attrs=c)
        return out[0], out[1], out[2], out[4] if c is not None else None, out[3]
    return fn


def assert_matches_fixture(z, tag, verts, faces, L, vc, keys, grads, atol=1e-5, grtol=1e-4):
    """Mesh up to relabelling (faces exactly; vertices, L_dev and colours within atol) and gradients within grtol of
    each tensor's largest magnitude, zero off the surface, against the fixture entry `tag`
    ("case/ws/given/colours/training"; the geometry is stored under the colours-given tag)."""
    name, ws, given, _, training = tag.split("/")
    geo = f"{name}/{ws}/{given}/1/{training}"
    rk = tuple(torch.from_numpy(z[f"{geo}/{k}"]).long() for k in ("vkeys", "lvkeys", "ledges"))
    RV, RF, RL = O.canonical(torch.from_numpy(z[geo + "/verts"]), torch.from_numpy(z[geo + "/faces"]).long(),
                             torch.from_numpy(z[geo + "/L"]), rk)
    V, Fs, Ld = O.canonical(verts.double().cpu(), faces.cpu(), L.double().cpu(), tuple(k.cpu() for k in keys))
    assert V.keys() == RV.keys(), (tag, len(V), len(RV))
    assert Fs == RF, (tag, len(Fs), len(RF), len(Fs ^ RF))
    assert Ld.keys() == RL.keys(), tag
    if V:
        dv = max(max(abs(a - b) for a, b in zip(V[k], RV[k])) for k in V)
        assert dv <= atol, (tag, "verts", dv)
    if Ld:
        dl = max(abs(Ld[k] - RL[k]) for k in Ld)
        assert dl <= atol, (tag, "L_dev", dl)
    assert (vc is None) == (tag + "/colours" not in z.files), tag
    if vc is not None:
        ref = torch.from_numpy(z[tag + "/colours"]).double()
        assert vc.shape == ref.shape, (tag, vc.shape, ref.shape)
        if ref.numel():
            C = {k: r for k, r in zip(rk[0].tolist(), ref)}
            got = {k: r for k, r in zip(keys[0].cpu().tolist(), vc.double().cpu())}
            dc = max(float((got[k] - C[k]).abs().max()) for k in C)
            assert dc <= atol, (tag, "colours", dc)
    if grads is None:
        assert tag + "/gx" not in z.files, tag
        return
    rows = torch.from_numpy(z[name + "/grows"]).long()
    names = []
    for n in ("gx", "gs", "gc"):
        g = grads.get(n)
        assert (g is None) == (f"{tag}/{n}" not in z.files), (tag, n)
        if g is None:
            continue
        g = g.cpu()
        rest = torch.ones(g.shape[0], dtype=torch.bool)
        rest[rows] = False
        assert not g[rest].any(), (tag, n, "off the surface")
        names.append((n, g[rows]))
    if grads.get("gw") is not None:
        wrows = torch.from_numpy(z[name + "/gw_rows"]).long()
        gw = grads["gw"].cpu()
        rest = torch.ones(gw.shape[0], dtype=torch.bool)
        rest[wrows] = False
        assert not gw[rest].any(), (tag, "weight gradient off the surface cubes")
        names.append(("gw", gw[wrows]))
    for n, g in names:
        ref = torch.from_numpy(z[f"{tag}/{n}"]).double()
        err = float((g.double() - ref).abs().max())
        scale = float(ref.abs().max())
        assert err <= grtol * max(scale, 1e-12), (tag, n, err, scale)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference(name, dtype):
    res, x, s, w, c = case_inputs(Z, name)
    for ws, given, colours, training in variants(name):
        v, f, L, vc, keys, grads = run_with_grads(oracle_fn(res, bool(training), ws, dtype), x, s, w, c, given,
                                                  colours, Z)
        assert_matches_fixture(Z, f"{name}/{ws}/{given}/{colours}/{training}", v, f, L, vc, keys, grads)


def test_fixture_covers_the_trellis_layout():
    """The trellis case has SparseFeatures2Mesh's dense layout: default sdf 1 and zero colours and weights off the
    sparse cubes, a surface, and quads."""
    res, x, s, w, c = case_inputs(Z, "trellis")
    assert res == (32, 32, 32) and c.shape == (33 ** 3, 6) and w.shape == (32 ** 3, 21)
    off = s == 1
    assert 0.5 < float(off.float().mean()) < 1 and not c[off].any()
    assert Z["trellis/0.99/1/1/0/faces"].shape[0] > 500


def test_no_fixture_case_has_zero_sdf():
    """No grid point sits at s == 0 exactly, where a group's |d_e - mean(d)| can sit at its kink and the subgradient
    depends on the last bits: so every case's gradients are held to 1e-4 of their largest magnitude."""
    for name in CASES:
        _, _, s, _, _ = case_inputs(Z, name)
        assert not (s == 0).any(), name


@pytest.mark.parametrize("res", [64, 256])
def test_closed_form_grid_matches_construct_dense_grid(res):
    """construct_dense_grid's cube_idx is voxel_grid's cube array, and its verts are the integer point coordinates
    in the same point order."""
    from gs_b200.isosurface import voxel_grid
    _, cubes = voxel_grid(res, "cpu")
    a = torch.arange(res + 1)
    verts = torch.stack(torch.meshgrid(a, a, a, indexing="ij"), -1).reshape(-1, 3)
    assert [verts.shape[0], cubes.shape[0]] == Z[f"dense_grid/{res}/shapes"].tolist()
    assert hashlib.sha256(verts.numpy().tobytes()).hexdigest() == Z[f"dense_grid/{res}/sha256"][0]
    assert hashlib.sha256(cubes.numpy().tobytes()).hexdigest() == Z[f"dense_grid/{res}/sha256"][1]
