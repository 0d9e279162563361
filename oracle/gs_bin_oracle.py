"""Exact restatement of the binning stage (csrc/gs_sort.cu, csrc/gs_binning.cu, bin_a / bin_b in csrc/gs_capi.cu), in
numpy integers.

Inputs are one view's integer preprocess outputs, which the tests pin separately to `gs_oracle.preprocess` bit for
bit: tiles_touched, the tile rect [x0, x1) x [y0, y1) of every Gaussian, its depth key (the fp32 bits of t.z, or
0xFFFFFFFF when it is culled) and, with tile culling, its per-row spans (4 x uint32: row r is the 16-bit entry
r of the 8 packed in the words, start = e & 255 and count = e >> 8, tiles x0 + start ... x0 + start + count - 1 of tile
row y0 + r; spans[0] = 0xFFFFFFFF means the whole square).

From those it gives the stable depth order (invisible Gaussians last, ties by index), the exclusive scan of
tiles_touched in that order, the (tile, Gaussian) lists in (tile, depth, index) order -- the package's full squares or
the culled rows -- and the per-tile ranges [start, end) ([0, 0] for an empty tile).
"""
import numpy as np

INVISIBLE = np.uint32(0xFFFFFFFF)


def depth_order(dkeys):
    """stable ascending order of the u32 depth keys: invisible (0xFFFFFFFF) last, ties by Gaussian index"""
    return np.argsort(np.asarray(dkeys, dtype=np.uint32), kind="stable").astype(np.uint32)


def scan(tiles, order):
    """exclusive prefix sums of tiles_touched in depth order (u32) and the view's total"""
    t = np.asarray(tiles, dtype=np.int64)[order]
    inc = np.cumsum(t)
    return (inc - t).astype(np.uint32), int(inc[-1]) if t.size else 0


def emit(order, tiles, rmin, rmax, gx, spans=None):
    """(tile key, Gaussian) pairs in depth order, each Gaussian's tiles row-major: its whole square, or (spans given
    and spans[i, 0] != 0xFFFFFFFF) the tiles of its decoded rows"""
    tiles = np.asarray(tiles, dtype=np.int64)
    ids = np.asarray(order, dtype=np.int64)
    ids = ids[tiles[ids] > 0]
    cnt = tiles[ids]
    total = int(cnt.sum())
    if total == 0:
        return np.empty(0, np.uint32), np.empty(0, np.uint32)
    rep = np.repeat(ids, cnt)
    local = np.arange(total, dtype=np.int64) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    x0, y0 = rmin[rep, 0].astype(np.int64), rmin[rep, 1].astype(np.int64)
    w = rmax[rep, 0].astype(np.int64) - x0
    ry, rx = local // w, local % w
    if spans is not None:
        sp = np.asarray(spans, dtype=np.uint32).reshape(-1, 4)
        tight = sp[rep, 0] != INVISIBLE
        if tight.any():
            s = sp[rep[tight]].astype(np.int64)
            rem = local[tight].copy()
            ty, tx = np.zeros_like(rem), np.zeros_like(rem)
            found = np.zeros(rem.shape, bool)
            for r in range(8):
                e = (s[:, r >> 1] >> (16 * (r & 1))) & 0xFFFF
                c, st = e >> 8, e & 255
                hit = ~found & (rem < c)
                ty[hit], tx[hit] = r, st[hit] + rem[hit]
                found |= hit
                rem = np.where(found, rem, rem - c)
            assert found.all(), "tiles_touched exceeds the decoded rows"
            ry[tight], rx[tight] = ty, tx
    keys = (y0 + ry) * gx + x0 + rx
    return keys.astype(np.uint32), rep.astype(np.uint32)


def tile_sort(keys, vals):
    """stable sort of the pairs by tile: (tile, depth, index) order"""
    o = np.argsort(keys, kind="stable")
    return keys[o], vals[o]


def ranges(sorted_keys, ntiles):
    """[ntiles, 2] u32: [start, end) of each tile in the sorted list, [0, 0] when the tile has no pair"""
    r = np.zeros((ntiles, 2), np.uint32)
    if sorted_keys.size == 0:
        return r
    k = sorted_keys.astype(np.int64)
    change = np.nonzero(np.diff(k))[0] + 1
    starts = np.concatenate([[0], change])
    ends = np.concatenate([change, [k.size]])
    r[k[starts], 0] = starts
    r[k[starts], 1] = ends
    return r


def bin_view(dkeys, tiles, rmin, rmax, gx, gy, spans=None):
    """everything the binning of one view computes; spans=None gives the package's lists"""
    order = depth_order(dkeys)
    offsets, total = scan(tiles, order)
    keys, vals = tile_sort(*emit(order, tiles, rmin, rmax, gx, spans))
    assert keys.size == total
    return dict(order=order, sorted_dkeys=np.asarray(dkeys, np.uint32)[order], offsets=offsets, total=total,
                tile_keys=keys, point_list=vals, ranges=ranges(keys, gx * gy))
