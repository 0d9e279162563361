"""CPU half of the binning edge suite (tests/test_gpu_binning_edges.py): the exact binning oracle pinned to the package's
64-bit-key restatement in `gs_oracle`, and the premise of every GPU scene checked on the CPU -- that the scene
reaches the edge it is named for."""
import numpy as np
import pytest
import torch

from oracle import gs_bin_oracle as BO
from oracle import gs_oracle as O
import test_gpu_binning_edges as S

f32 = np.float32


def test_oracle_matches_package_restatement():
    """the package's lists: (tile << 32 | depth) keys emitted by Gaussian index, one stable 64-bit sort -- equal to the
    depth sort, the emit in depth order and the stable tile sort of the binning oracle"""
    for seed, (W, H) in enumerate([(128, 128), (272, 144), (40, 24)]):
        cl = S.cloud(3000, seed=seed, ties=seed == 1)
        st = S.settings(W, H)
        pre = S.pre(cl, st)
        keys, vals = O.sort_pairs(*O.duplicate_with_keys(pre))
        ref_ranges = O.identify_tile_ranges(keys, pre["grid"][0] * pre["grid"][1])
        got = S.oracle_view(pre, None)
        assert np.array_equal(got["point_list"], vals)
        assert np.array_equal(got["tile_keys"].astype(np.uint64), keys >> np.uint64(32))
        assert np.array_equal(got["ranges"], ref_ranges)
        assert got["total"] == keys.size


def test_oracle_culled_rows():
    """whole-square spans give the package's lists; decoded rows give exactly the listed tiles, row-major"""
    rmin = np.array([[2, 1], [0, 0]]); rmax = np.array([[6, 4], [2, 1]])
    tiles = np.array([5, 2]); gx = 8
    sp = np.zeros((2, 4), np.uint32)
    sp[0, 0] = (1 | (2 << 8)) | ((0 | (3 << 8)) << 16)       # row 0: x0+1, x0+2; row 1: x0 .. x0+2
    sp[1, 0] = 0xFFFFFFFF
    k, v = BO.emit(np.array([1, 0]), tiles, rmin, rmax, gx, sp)
    assert k.tolist() == [0, 1, 1 * gx + 3, 1 * gx + 4, 2 * gx + 2, 2 * gx + 3, 2 * gx + 4]
    assert v.tolist() == [1, 1, 0, 0, 0, 0, 0]
    full = np.array([[0xFFFFFFFF, 0, 0, 0]] * 2, np.uint32)
    area = (rmax - rmin).prod(1)
    assert np.array_equal(np.stack(BO.emit(np.array([0, 1]), area, rmin, rmax, gx, full)),
                          np.stack(BO.emit(np.array([0, 1]), area, rmin, rmax, gx, None)))
    r = BO.ranges(np.array([0, 0, 3, 3, 3], np.uint32), 5)
    assert r.tolist() == [[0, 2], [0, 0], [0, 0], [2, 5], [0, 0]]


def test_b1_premise_depth_keys():
    """t.z of the near-plane pair is exactly 0.2f and one ulp above; the tie cloud has many equal depth keys; the far
    splat makes the top digit of (key - min) non-trivial, the near cloud alone keeps it trivial"""
    st = S.b1_settings()
    cl = S.b1_cloud(4097, far=False)
    tz = S.pre(cl, st)["depth"].numpy().astype(f32)
    assert tz[0] == f32(0.2) and tz[1] == np.nextafter(f32(0.2), f32(1))
    pre = S.pre(cl, st)
    assert int(pre["radii"][0]) == 0 and int(pre["radii"][1]) > 0
    k = S.depth_keys(pre)
    vis = k[k != 0xFFFFFFFF]
    assert len(vis) - len(np.unique(vis)) > 1000
    assert (int(vis.max()) - int(vis.min())) >> 24 == 0
    kf = S.depth_keys(S.pre(S.b1_cloud(4097, far=True), st))
    kf = kf[kf != 0xFFFFFFFF]
    assert (int(kf.max()) - int(kf.min())) >> 24 > 0
    away = S.pre(cl, S.b1_settings(away=True))
    assert int(away["tiles_touched"].sum()) == 0


def test_b2_premise_scan_chunks():
    """the scan's block sums (2048 Gaussians a block) are carried over 1024-block chunks: 2^21 + 1 Gaussians need two,
    5 000 000 three; 131 587 full-frame 1080p splats make 2^30 pairs or more, 2^30 - 1 pairs fit"""
    chunks = lambda n: -(-(-(-n // 2048)) // 1024)        # noqa: E731
    assert [chunks(n) for n in S.B2_SIZES] == [1, 1, 1, 1, 1, 2, 3]
    tiles = 120 * 68
    assert 131587 * tiles >= 2 ** 30 > 131586 * tiles
    assert 131586 * tiles + S.LIMIT_SMALL == 2 ** 30 - 1


def test_b3_premise_span_limits():
    """the squares of the span scene are 255 and 256 tiles wide (4096 x 128) and 8 and 9 rows high (272 x 144), on
    both sides of tight_spans' whole-square limit; opacities straddle o * 255 >= 1"""
    for (W, H), axis, want in (((4096, 128), 0, {255, 256}), ((272, 144), 1, {8, 9})):
        pre = S.pre(S.b3_cloud(W, H), S.settings(W, H))
        ext = (pre["rect_max"] - pre["rect_min"]).numpy()[pre["radii"].numpy() > 0]
        assert want <= set(ext[:, axis].tolist())
        assert (ext[:, 0] <= 255).all() or axis == 0
    o = S.b3_cloud(272, 144)["opacities"].astype(f32).ravel()
    assert (o * f32(255) < 1).any() and ((o * f32(255) >= 1) & (o < f32(0.01))).any()


def test_b4_premise_tile_sort_passes():
    """1, 256, 272, 65 536 and 65 792 tiles: the tile sort's key width needs 1, 1, 2, 2 and 3 digit passes"""
    bits = lambda n: max(1, int(np.ceil(np.log2(n))))     # noqa: E731  (bits_for in gs_capi.cu)
    tiles = [((W + 15) // 16) * ((H + 15) // 16) for W, H in S.B4_SIZES]
    assert tiles == [1, 256, 272, 65536, 65792]
    assert [-(-bits(t) // 8) for t in tiles] == [1, 1, 2, 2, 3]


def test_b6_premise_nan_extent():
    """Before the cull, a NaN extent became radius 0 with a one-tile rect: the scan reserved one slot, the emit (radius
    > 0 only) filled none.  Restated on the preprocess's integer path (PTX cvt.rzi of NaN is 0)."""
    st = S.settings(128, 96, azim=30.0, elev=20.0)
    cl = S.b6_cloud()
    pre = S.pre(cl, st)
    radf = S.extent32(cl, st)
    bad = S.B6_BAD
    assert np.isnan(radf[bad]).any() and np.isinf(radf[bad]).any()
    xy = pre["xy"].detach().numpy().astype(f32)
    gx, gy = pre["grid"]
    for i in np.nonzero(np.isnan(radf))[0]:
        rad_i = 0                                             # (int)NaN
        x0 = min(gx, max(0, int((xy[i, 0] - f32(rad_i)) / f32(16))))
        x1 = min(gx, max(0, int((xy[i, 0] + f32(rad_i) + f32(15)) / f32(16))))
        y0 = min(gy, max(0, int((xy[i, 1] - f32(rad_i)) / f32(16))))
        y1 = min(gy, max(0, int((xy[i, 1] + f32(rad_i) + f32(15)) / f32(16))))
        scan_count = (x1 - x0) * (y1 - y0)
        emit_count = scan_count if rad_i > 0 else 0
        assert (scan_count, emit_count) == (1, 0)
        assert int(pre["radii"][i]) == 0 and int(pre["tiles_touched"][i]) == 0      # the oracle culls it
    for i in np.nonzero(np.isinf(radf))[0]:
        assert int(pre["radii"][i]) == 2 ** 31 - 1 and int(pre["tiles_touched"][i]) == gx * gy
    pc = S.pre(S.b6_cov_cloud(), S.settings(128, 96, azim=30.0, elev=20.0))
    r = pc["radii"].numpy()
    assert r[S.B6_COV_BAD[0]] == 0 and r[S.B6_COV_BAD[1]] > 0 and (r[:S.B6_COV_BAD[0]] > 0).any()


def test_b7_premise_segments():
    """the direct sort's segment sets have empty segments first, middle and last and lengths 4096 +- 1"""
    sets = S.b7_cases()
    lens = [np.diff(c["off"]).tolist() for c in sets]
    assert any(l[0] == 0 for l in lens) and any(l[-1] == 0 for l in lens) and any(0 in l[1:-1] for l in lens)
    assert {4095, 4096, 4097, 12289} <= set(sum(lens, []))
    assert max(len(l) for l in lens) == 16 and min(len(l) for l in lens) == 1


@pytest.mark.parametrize("case", range(len(S.b7_cases())))
def test_b7_oracle_is_stable_argsort(case):
    c = S.b7_cases()[case]
    k, v = S.b7_oracle(c)
    for i in range(len(c["off"]) - 1):
        a, b = c["off"][i], c["off"][i + 1]
        kk = S.b7_digits(c, i, c["keys"][a:b])
        assert np.all(np.diff(S.b7_digits(c, i, k[a:b]).astype(np.int64)) >= 0)
        assert sorted(v[a:b].tolist()) == list(range(a, b))
        assert np.array_equal(kk[v[a:b] - a], S.b7_digits(c, i, k[a:b]))
