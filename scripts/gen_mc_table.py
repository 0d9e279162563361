"""Derives the marching-cubes case table and writes comfyui-3d-pack_b200/csrc/mc_table.cuh.

    python scripts/gen_mc_table.py            # rewrite the header
    python scripts/gen_mc_table.py --check    # exit 1 if the committed header differs

Numbering (shared with csrc/ngp_mcubes.cu and oracle/mc_oracle.py):
- corner i of a cell sits at offset (i & 1, (i >> 1) & 1, (i >> 2) & 1) along array axes (0, 1, 2) from the cell's
  min corner; bit i of the cube index is set iff that corner's value > iso ("above").
- edge e = 4 * a + k runs along axis a from the corner with a-offset 0 to the one with a-offset 1; the offsets along
  the other two axes b < c are (k & 1, k >> 1).
- an edge crosses iff exactly one of its ends is above.

The triangulation is derived, not transcribed:
1. On each of the 6 faces the crossing edges (0, 2 or 4 of them) are joined into segments. With 4 (diagonal corners
   alike) each segment cuts off one ABOVE corner. The rule reads only the face's own four signs, so the two cells
   sharing a face draw the same segments there and the mesh is watertight.
2. Each segment is oriented along g x f, where f is the face's outward normal and g the in-face direction from the
   segment's above side to its below side. That is the boundary orientation (Stokes) of a surface whose normal
   points from above to below.
   The two cells sharing a face see opposite f, so they traverse each shared segment in opposite directions.
3. The oriented segments form closed loops (every crossing edge lies on two faces: one segment leaves it, one enters).
   Loops are taken in order of their lowest edge, and each loop is fanned from its lowest edge.
Triangles are therefore counter-clockwise seen from the below-iso side: the right-hand normal points from above to
below, outward for a density blob.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "comfyui-3d-pack_b200", "csrc", "mc_table.cuh")
PAD = 255


def corner_pos(i):
    return np.array([i & 1, (i >> 1) & 1, (i >> 2) & 1], dtype=np.float64)


def edge_corners(e):
    """(low corner, high corner) of edge e."""
    a, k = divmod(e, 4)
    b, c = [x for x in range(3) if x != a]
    base = (((k & 1) << b) | ((k >> 1) << c))
    return base, base | (1 << a)


def edge_mid(e):
    lo, hi = edge_corners(e)
    return 0.5 * (corner_pos(lo) + corner_pos(hi))


FACES = [(a, s) for a in range(3) for s in range(2)]


def face_corners(a, s):
    return [i for i in range(8) if ((i >> a) & 1) == s]


def face_edges(a, s):
    out = []
    for e in range(12):
        lo, hi = edge_corners(e)
        if e // 4 != a and ((lo >> a) & 1) == s and ((hi >> a) & 1) == s:
            out.append(e)
    return out


def above(cube, i):
    return (cube >> i) & 1 == 1


def crossing_edges(cube):
    return [e for e in range(12) if above(cube, edge_corners(e)[0]) != above(cube, edge_corners(e)[1])]


def face_segments(cube, a, s):
    """Oriented segments (e_from, e_to) that the face (a, s) contributes to the cell's boundary loops."""
    corners = face_corners(a, s)
    f = np.zeros(3); f[a] = 2 * s - 1
    cross = [e for e in face_edges(a, s) if e in crossing_edges(cube)]
    raw = []                                   # (e1, e2, g)
    if len(cross) == 2:
        A = [corner_pos(i) for i in corners if above(cube, i)]
        B = [corner_pos(i) for i in corners if not above(cube, i)]
        raw.append((cross[0], cross[1], np.mean(B, axis=0) - np.mean(A, axis=0)))
    elif len(cross) == 4:
        centre = np.mean([corner_pos(i) for i in corners], axis=0)
        for c in corners:
            if above(cube, c):
                es = [e for e in cross if c in edge_corners(e)]
                assert len(es) == 2
                raw.append((es[0], es[1], centre - corner_pos(c)))
    else:
        assert not cross
    segs = []
    for e1, e2, g in raw:
        d = np.cross(g, f)
        if np.dot(edge_mid(e2) - edge_mid(e1), d) < 0:
            e1, e2 = e2, e1
        segs.append((e1, e2))
    return segs


def cell_segments(cube):
    return [sg for a, s in FACES for sg in face_segments(cube, a, s)]


def cell_triangles(cube):
    nxt = {}
    for e1, e2 in cell_segments(cube):
        assert e1 not in nxt, (cube, e1)
        nxt[e1] = e2
    assert sorted(nxt) == sorted(nxt.values()) == crossing_edges(cube), cube
    tris, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e); loop.append(e); e = nxt[e]
        assert e == start and len(loop) >= 3, (cube, loop)
        # start is the loop's lowest edge: loops are entered in increasing order of their lowest edge
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


def build_table():
    tables = [cell_triangles(c) for c in range(256)]
    max_tris = max(len(t) for t in tables)
    # The kernels and the oracle size their per-cell buffers from MC_MAX_TRIS; a change of rule that changes it
    # has to be looked at, not absorbed silently.
    assert max_tris == 5, max_tris
    return tables, max_tris


def render(tables, max_tris):
    lines = [
        "// Marching-cubes case table. Generated by scripts/gen_mc_table.py; do not edit.",
        "// Corner i is at offset (i & 1, (i >> 1) & 1, (i >> 2) & 1) from the cell's min corner; cube index bit i = value > iso.",
        "// Edge e = 4 * a + k runs along axis a; its offsets along the other two axes b < c are (k & 1, k >> 1).",
        "// Triangles are counter-clockwise seen from the below-iso side; unused entries are 255.",
        "#pragma once",
        "",
        f"#define MC_MAX_TRIS {max_tris}",
        "",
        "static __device__ const unsigned char mc_tri_count[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(tables[c])) for c in range(r, r + 32)) + ",")
    lines.append("};")
    lines.append("")
    lines.append("static __device__ const unsigned char mc_tri_edges[256][3 * MC_MAX_TRIS] = {")
    for c in range(256):
        flat = [e for t in tables[c] for e in t] + [PAD] * (3 * (max_tris - len(tables[c])))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "},")
    lines.append("};")
    return "\n".join(lines) + "\n"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--check", action="store_true", help="compare with the committed header instead of writing it")
    ap.add_argument("--out", default=HEADER)
    args = ap.parse_args()
    text = render(*build_table())
    if args.check:
        ok = os.path.exists(args.out) and open(args.out).read() == text
        print("mc_table.cuh is up to date" if ok else "mc_table.cuh differs from the generator's output")
        sys.exit(0 if ok else 1)
    with open(args.out, "w") as fh:
        fh.write(text)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
