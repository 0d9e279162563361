"""Marching cubes without a GPU: the case table (scripts/gen_mc_table.py -> csrc/mc_table.cuh) and the numpy oracle
(oracle/mc_oracle.py) that tests/test_gpu_mcubes.py compares the kernels against bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import mc_oracle as M

sys.path.insert(0, os.path.join(ROOT, "scripts"))
import gen_mc_table as G  # noqa: E402

COUNTS, EDGES = M.load_table()


def _tris(cube):
    return [tuple(int(e) for e in EDGES[cube, 3 * i:3 * i + 3]) for i in range(COUNTS[cube])]


def _above(cube, i):
    return (cube >> i) & 1 == 1


def _crossing(cube):
    return {e for e in range(12) if _above(cube, G.edge_corners(e)[0]) != _above(cube, G.edge_corners(e)[1])}


def _face_rule_segments(cube):
    """Undirected face segments by the rule, derived here from the face signs alone: 2 crossing edges are joined;
    with 4, each above corner is cut off by the two crossing edges that meet at it."""
    segs = set()
    for a in range(3):
        for s in range(2):
            corners = [i for i in range(8) if ((i >> a) & 1) == s]
            fe = [e for e in _crossing(cube) if e // 4 != a and all(((c >> a) & 1) == s for c in G.edge_corners(e))]
            if len(fe) == 2:
                segs.add(frozenset(fe))
            elif len(fe) == 4:
                for c in corners:
                    if _above(cube, c):
                        segs.add(frozenset(e for e in fe if c in G.edge_corners(e)))
            else:
                assert not fe
    return segs


def test_generator_reproduces_the_committed_header(tmp_path):
    out = tmp_path / "mc_table.cuh"
    subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gen_mc_table.py"), "--out", str(out)], check=True,
                   capture_output=True)
    with open(G.HEADER, "rb") as fh:
        assert out.read_bytes() == fh.read()


def test_table_size_and_padding():
    assert EDGES.shape[1] == 3 * int(COUNTS.max())
    for c in range(256):
        assert (EDGES[c, 3 * COUNTS[c]:] == G.PAD).all()
    assert COUNTS[0] == 0 and COUNTS[255] == 0


@pytest.mark.parametrize("cube", range(256))
def test_table_case(cube):
    tris = _tris(cube)
    # only crossing edges, and every crossing edge
    assert {e for t in tris for e in t} == _crossing(cube)
    directed = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
    assert len(set(directed)) == len(directed)
    # interior edges occur twice, once in each direction; the rest is the boundary
    boundary = [d for d in directed if (d[1], d[0]) not in directed]
    interior = [d for d in directed if (d[1], d[0]) in directed]
    assert len(interior) % 2 == 0
    # the boundary of the cell's triangles is exactly its face segments
    assert {frozenset(d) for d in boundary} == _face_rule_segments(cube)
    assert len(boundary) == len(_face_rule_segments(cube))
    # each loop (the fan from its lowest edge) faces its below corners: its vector area, with edge-midpoint
    # vertices, has a positive component along the sum of its edges' (below end - above end)
    loops = {}
    for t in tris:
        assert t[0] == min(t)
        loops.setdefault(t[0], []).append(t)
    for fan in loops.values():
        area = sum(np.cross(G.edge_mid(t[1]) - G.edge_mid(t[0]), G.edge_mid(t[2]) - G.edge_mid(t[0])) for t in fan)
        toward_below = 0
        for e in {e for t in fan for e in t}:
            lo, hi = G.edge_corners(e)
            a, b = (lo, hi) if _above(cube, lo) else (hi, lo)
            toward_below = toward_below + G.corner_pos(b) - G.corner_pos(a)
        assert np.dot(area, toward_below) > 0


# ---- oracle ----------------------------------------------------------------------------------------------------
def test_one_corner_above_gives_one_triangle_at_the_interpolated_positions():
    vol = np.zeros((2, 2, 2), np.float32)
    vol[0, 0, 0] = 1.0
    v, t = M.marching_cubes(vol, 0.25)            # t = (0.25 - 1) / (0 - 1) = 0.75 along each edge of corner 0
    assert v.dtype == np.float32 and t.dtype == np.int32
    assert np.array_equal(v, np.array([[0.75, 0, 0], [0, 0.75, 0], [0, 0, 0.75]], np.float32))
    assert np.array_equal(t, np.array([[0, 1, 2]], np.int32))
    n = M.triangle_normals(v, t)[0]
    assert (n > 0).all()                          # away from the above corner (0,0,0)


def test_ambiguous_face_separates_the_above_corners():
    vol = np.zeros((2, 2, 2), np.float32)
    vol[0, 0, 0] = vol[1, 1, 0] = 1.0             # diagonal above corners on the face z = 0
    v, t = M.marching_cubes(vol, 0.5)
    assert t.shape == (2, 3)
    assert not set(t[0]) & set(t[1])
    cut = []
    for tri in t:
        # each triangle's vertices lie half way along the three edges of one above corner
        corner = next(c for c in (np.array([0, 0, 0]), np.array([1, 1, 0]))
                      if np.array_equal(np.abs(v[tri] - c).sum(axis=1), [0.5, 0.5, 0.5]))
        cut.append(tuple(corner))
        n = M.triangle_normals(v, tri[None])[0]
        assert np.dot(n, v[tri].mean(axis=0) - corner) > 0
    assert sorted(cut) == [(0, 0, 0), (1, 1, 0)]


def _grid(n):
    return np.indices((n, n, n)).astype(np.float64).transpose(1, 2, 3, 0)


def test_sphere_is_a_closed_outward_sphere():
    n, r, c = 64, 24.3, np.array([31.7, 32.2, 31.9])
    vol = (r - np.linalg.norm(_grid(n) - c, axis=-1)).astype(np.float32)
    v, t = M.marching_cubes(vol, 0.0)
    assert M.is_oriented_manifold(t)
    assert M.euler_characteristic(len(v), t) == 2
    nrm = M.triangle_normals(v, t)
    assert (np.einsum("ij,ij->i", nrm, v[t].mean(axis=1) - c) > 0).all()
    assert abs(M.signed_volume(v, t) / (4 / 3 * np.pi * r ** 3) - 1) < 0.01


def test_torus_has_euler_characteristic_zero():
    n, R, r = 64, 20.0, 7.3
    p = _grid(n) - np.array([31.6, 32.1, 31.8])
    vol = (r - np.sqrt((np.hypot(p[..., 0], p[..., 1]) - R) ** 2 + p[..., 2] ** 2)).astype(np.float32)
    v, t = M.marching_cubes(vol, 0.0)
    assert M.is_oriented_manifold(t)
    assert M.euler_characteristic(len(v), t) == 0


@pytest.mark.parametrize("seed,shape", [(0, (9, 10, 11)), (1, (16, 16, 16)), (2, (5, 23, 7)), (3, (2, 2, 40))])
def test_random_fields_bordered_below_iso_are_closed_and_oriented(seed, shape):
    rng = np.random.default_rng(seed)
    vol = rng.uniform(-1, 1, shape).astype(np.float32)
    vol[[0, -1], :, :] = vol[:, [0, -1], :] = vol[:, :, [0, -1]] = -1.0
    v, t = M.marching_cubes(vol, 0.0)
    if min(shape) > 2:
        assert len(t) > 0
    # Closed and consistently oriented.  Not always a manifold: a cell loop that crosses one face twice can be fanned
    # into a triangle lying in that face, and the neighbour across it then fans the same triangle reversed.
    assert M.is_closed_oriented(t)
    assert t.min(initial=0) >= 0 and t.max(initial=-1) < len(v)
    assert len(np.unique(t)) == len(v)            # every vertex is used


def test_slabs_do_not_change_the_result():
    vol = np.random.default_rng(4).uniform(-1, 1, (21, 8, 9)).astype(np.float32)
    ref = M.marching_cubes(vol, 0.1, slab=64)
    for slab in (1, 2, 5):
        got = M.marching_cubes(vol, 0.1, slab=slab)
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])


def test_degenerate_and_non_finite_volumes():
    for shape in ((1, 5, 5), (5, 1, 5), (5, 5, 1), (0, 4, 4)):
        v, t = M.marching_cubes(np.ones(shape, np.float32), 0.5)
        assert v.shape == (0, 3) and t.shape == (0, 3)
    vol = np.zeros((4, 4, 4), np.float32)
    vol[1, 2, 3] = np.nan
    with pytest.raises(ValueError, match="non-finite"):
        M.marching_cubes(vol, 0.5)


def test_mcubes_shim_surface_without_a_device():
    import mcubes
    for name in ("smooth", "export_obj", "marching_cubes_func"):
        with pytest.raises(NotImplementedError):
            getattr(mcubes, name)(np.zeros((2, 2, 2)))
    with pytest.raises(TypeError):
        mcubes.marching_cubes(np.zeros((2, 2, 2), np.complex64), 0.0)
    with pytest.raises(ValueError):
        mcubes.marching_cubes(np.zeros((2, 2), np.float32), 0.0)
