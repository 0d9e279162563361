"""Binning (csrc/gs_sort.cu, csrc/gs_binning.cu, bin_a / bin_b in csrc/gs_capi.cu) against the exact integer oracle
`oracle/gs_bin_oracle.py`, at the edges where it goes wrong: the depth sort's ties, near plane, empty and one-splat
views and trivial digits (B1), the scan's block-sum carry and the per-view pair limit (B2), the emit's zero-count
warps, whole-square and culled spans at tight_spans' 255-wide / 8-row limits and the 1/255 opacity edge (B3), the tile
sort at 1 to 3 digit passes (B4), the step's view chunks with empty views and 4096 +- 1 Gaussians (B5), Gaussians
whose extent is NaN or infinite (B6), and the segmented sort itself (B7).  Every scene has a CPU test of its premise
in tests/test_binning_edges_cpu.py.

The lists are the ones the multi-view step walks: `gs_b200_debug_bin_views` runs the step's own chunking, batched
preprocess, depth sort, scan, view_spans and emit / tile sort / ranges, with tile culling on or off, and returns every
intermediate.  Its pair buffers are filled with 0xFFFFFFFF before the emit, so an unwritten slot shows.  Radii, tiles
and rects must equal `gs_oracle.preprocess`'s; depth order, offsets, lists and ranges the exact oracle's; every view's
lists must count each Gaussian tiles_touched times, hold only keys below the tile count, and its ranges partition its
pairs.  A second run must be bit-identical."""
import ctypes as C
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import gs_bin_oracle as BO
from oracle import gs_oracle as O

f32 = np.float32
FOVY = 49.1
SENT = 0xFFFFFFFF


# ---------------------------------------------------------------------------------------------------------------------
# scenes (shared with the CPU premise tests)
# ---------------------------------------------------------------------------------------------------------------------
def settings(W, H, away=False, radius=1.75, azim=0.0, elev=0.0):
    if away:        # looks along +z from z = 1.75: every Gaussian of the unit ball is behind the camera
        c2w = O.orbit_camera(0.0, 180.0, 1.75, target=np.array([0, 0, 3.5], f32))
    else:
        c2w = O.orbit_camera(elev, azim, radius)
    return O.minicam_settings(c2w, W, H, FOVY)


def cloud(n, seed=0, ties=False, scale=0.02):
    rng = np.random.RandomState(seed)
    xyz = rng.uniform(-0.5, 0.5, (n, 3)).astype(f32)
    if ties:
        xyz[:, 2] = np.round(xyz[:, 2] * 8) / 8          # 9 depth levels: thousands of equal keys
    q = rng.normal(size=(n, 4))
    return dict(means3D=xyz, scales=np.exp(rng.normal(np.log(scale), 0.5, (n, 3))).astype(f32),
                rotations=(q / np.linalg.norm(q, axis=1, keepdims=True)).astype(f32),
                opacities=(1 / (1 + np.exp(-rng.normal(0, 2, (n, 1))))).astype(f32), shs=np.zeros((n, 1, 3), f32))


def pre(cl, st):
    t = lambda k: None if cl.get(k) is None else torch.as_tensor(cl[k])           # noqa: E731
    shs = t("shs") if cl.get("shs") is not None else torch.zeros(len(cl["means3D"]), 1, 3)
    return O.preprocess(t("means3D"), t("scales"), t("rotations"), t("opacities"), shs, None, t("cov3D_precomp"),
                        None, st)


def depth_keys(p):
    tz = p["depth"].detach().numpy().astype(f32).view(np.uint32)
    return np.where(p["radii"].numpy() > 0, tz, np.uint32(SENT)).astype(np.uint32)


def oracle_view(p, spans, tiles=None):
    gx, gy = p["grid"]
    t = p["tiles_touched"].numpy() if tiles is None else tiles
    return BO.bin_view(depth_keys(p), t, p["rect_min"].numpy(), p["rect_max"].numpy(), gx, gy, spans)


def near_plane_z(st, tz_want):
    """world z on the optical axis whose fp32 t.z is tz_want exactly (x = y = 0)"""
    m = st.viewmatrix.numpy().astype(f32).reshape(16)
    tz = lambda z: ((m[2] * f32(0) + m[6] * f32(0)) + m[10] * f32(z)) + m[14]        # noqa: E731
    z = f32((float(tz_want) - float(m[14])) / float(m[10]))
    for _ in range(400):
        d = tz(z)
        if d == tz_want:
            return z
        z = np.nextafter(z, f32(np.inf) if (d > tz_want) == (m[10] < 0) else f32(-np.inf))
    raise AssertionError("no z gives the wanted t.z")


def b1_settings(away=False):
    """close enough (0.45) that t.z = 0.45 - z can be 0.2f exactly"""
    return settings(128, 128, away=True) if away else settings(128, 128, radius=0.45)


def b1_cloud(n, far, seed=1):
    cl = cloud(n, seed=seed, ties=True)
    cl["means3D"][:, :2] *= 0.2
    cl["means3D"][:, 2] = cl["means3D"][:, 2] / 5 + f32(0.1)      # t.z in [0.25, 0.45]: a trivial top depth digit
    st = b1_settings()
    if n >= 3:
        for i, tzw in enumerate((f32(0.2), np.nextafter(f32(0.2), f32(1)))):
            cl["means3D"][i] = (0, 0, near_plane_z(st, tzw))
            cl["scales"][i] = 0.01
    if far:
        cl["means3D"][-1] = (0, 0, -40)
    return cl


B2_SIZES = [2047, 2048, 2049, 2 ** 21 - 1, 2 ** 21, 2 ** 21 + 1, 5_000_000]
LIMIT_SMALL = 2 ** 30 - 1 - 131586 * 8160


def small_cloud(n, seed=2, spread=0.9, tz=(1.3, 2.2), scale=2e-3):
    """n Gaussians of a few pixels spread over the frame of settings(W, H)"""
    rng = np.random.RandomState(seed)
    z = rng.uniform(1.75 - tz[1], 1.75 - tz[0], n).astype(f32)
    d = 1.75 - z
    t = np.tan(np.deg2rad(FOVY) / 2)
    xy = rng.uniform(-spread, spread, (n, 2)) * t * d[:, None]
    rot = np.zeros((n, 4), f32); rot[:, 0] = 1
    return dict(means3D=np.concatenate([xy, z[:, None]], 1).astype(f32), scales=np.full((n, 3), scale, f32),
                rotations=rot, opacities=np.full((n, 1), 0.5, f32), shs=np.zeros((n, 1, 3), f32))


def _concat(*cls):
    return {k: np.concatenate([c[k] for c in cls]) for k in cls[0]}


@lru_cache(maxsize=None)
def b3_cloud(W, H):
    """squares at tight_spans' limits (255 / 256 tiles wide at 4096 x 128, 8 / 9 rows high at 272 x 144), found by a
    search over the oracle's rects; opacities at 1/255 and one ulp either side; 64 zero-count splats adjacent in
    depth, then zero and non-zero counts mixed; needles"""
    st = settings(W, H)
    tx, ty = st.tanfovx * 1.75, st.tanfovy * 1.75
    if W > 1000:
        ss, xs, ys = np.linspace(7.4, 9.4, 41), np.linspace(-0.02, 0.02, 9) * tx, [0.0]
        pick = lambda w, h: w in (255, 256)           # noqa: E731
    else:
        ss, xs, ys = np.linspace(0.15, 0.45, 31), np.linspace(-0.3, 0.3, 7) * tx, np.linspace(-0.3, 0.3, 7) * ty
        pick = lambda w, h: h in (8, 9)               # noqa: E731
    g = np.array([(s, x, y) for s in ss for x in xs for y in ys], f32)
    n = len(g)
    cand = dict(means3D=np.stack([g[:, 1], g[:, 2], np.zeros(n, f32)], 1), scales=np.repeat(g[:, :1], 3, 1),
                rotations=np.tile(np.array([1, 0, 0, 0], f32), (n, 1)), opacities=np.full((n, 1), 0.8, f32),
                shs=np.zeros((n, 1, 3), f32))
    p = pre(cand, st)
    wh = (p["rect_max"] - p["rect_min"]).numpy()
    chosen, seen = [], {}
    for i in range(n):
        key = (int(wh[i, 0]), int(wh[i, 1]))
        if p["radii"][i] > 0 and pick(*key) and seen.get(key, 0) < 2:
            seen[key] = seen.get(key, 0) + 1
            chosen.append(i)
    big = {k: v[chosen] for k, v in cand.items()}
    rng = np.random.RandomState(3)
    o255 = f32(1) / f32(255)
    edge = small_cloud(6, seed=4, scale=0.05)
    edge["opacities"][:, 0] = [np.nextafter(o255, f32(0)), o255, np.nextafter(o255, f32(1))] * 2
    zero = small_cloud(64, seed=5, tz=(1.0, 1.02), scale=0.03)
    zero["opacities"][:] = 1e-3
    mixed = small_cloud(96, seed=6, tz=(1.1, 1.2), scale=0.03)
    mixed["opacities"][::2] = rng.choice([0.0, 1e-3, 0.5, 0.99], (48, 1)).astype(f32)
    needle = small_cloud(16, seed=7, scale=0.002)
    needle["scales"][:, 0] = 0.4
    a = rng.uniform(0, np.pi, 16)
    needle["rotations"] = np.stack([np.cos(a / 2), 0 * a, 0 * a, np.sin(a / 2)], 1).astype(f32)
    return _concat(big, edge, zero, mixed, needle)


B4_SIZES = [(16, 16), (256, 256), (272, 256), (4096, 4096), (4112, 4096)]

B6_BAD = [64, 65, 66, 67, 68]


def b6_cloud():
    """64 ordinary Gaussians, then: an infinite scale with an axis-aligned quaternion (0 * inf: NaN covariance), a scale
    of 2e19 (s^2 overflows), a NaN scale, a NaN quaternion, and an infinite scale with a general quaternion"""
    cl = small_cloud(64, seed=8, scale=0.03)
    bad = small_cloud(5, seed=9, scale=0.03)
    bad["scales"][0] = [np.inf, 0.03, 0.03]
    bad["scales"][1] = [2e19, 0.03, 0.03]
    bad["scales"][2] = [np.nan, 0.03, 0.03]
    bad["rotations"][3] = [np.nan, 0, 0, 0]
    bad["scales"][4] = [np.inf, np.inf, 0.03]
    bad["rotations"][4] = np.array([0.9, 0.3, 0.2, 0.1], f32) / np.linalg.norm([0.9, 0.3, 0.2, 0.1])
    return _concat(cl, bad)


B6_COV_BAD = [64, 65]


def b6_cov_cloud():
    """64 ordinary Gaussians as precomputed covariances, then a negative-definite one (culled) and an indefinite one
    (kept: its 2D covariance has one positive eigenvalue)"""
    cl = small_cloud(64, seed=10, scale=0.03)
    s = cl.pop("scales").astype(np.float64)[:, 0] ** 2
    cov = np.zeros((66, 6), f32)
    cov[:64, 0] = cov[:64, 3] = cov[:64, 5] = s
    cov[64] = [-0.01, 0, 0, -0.01, 0, -0.01]
    cov[65] = [0.01, 0, 0, -0.01, 0, 0.01]
    ex = small_cloud(2, seed=11)
    ex.pop("scales")
    out = _concat(cl, ex)
    out.pop("rotations")
    out["cov3D_precomp"] = cov
    return out


def extent32(cl, st):
    """ceil(3 sqrt(max eigenvalue)) of the fp32 2D covariance, with fmaxf's NaN rule, as project_view computes it"""
    ca, cb, cc = pre(cl, st)["cov2d"].detach().numpy().astype(f32).T
    with np.errstate(all="ignore"):
        det = ca * cc - cb * cb
        mid = f32(0.5) * (ca + cc)
        disc = np.sqrt(np.fmax(mid * mid - det, f32(0.1)))
        return np.ceil(f32(3) * np.sqrt(np.fmax(mid + disc, mid - disc)))


@lru_cache(maxsize=None)
def b7_cases():
    rng = np.random.RandomState(12)
    cases = []

    def add(lens, begin, end, bias=False, stride=1, gen=None):
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        nseg, n = len(lens), int(off[-1])
        b = rng.randint(0, 2 ** 32, nseg, dtype=np.uint64).astype(np.uint32) if bias else np.zeros(nseg, np.uint32)
        span = 1 << (begin + 8 * -(-(end - begin) // 8))
        keys = np.empty(n, np.uint32)
        for i in range(nseg):
            a, e = off[i], off[i + 1]
            k = rng.randint(0, min(span, 2 ** 32), e - a, dtype=np.uint64) if gen is None else gen(e - a)
            keys[a:e] = (k.astype(np.uint64) + b[i]) % 2 ** 32
            if bias and e - a > 4:
                keys[a:a + 2] = b[i]                  # keys equal to the bias: digit 0
                keys[a + 2] = SENT                    # 0xFFFFFFFF - bias: wraps like any other key
        cases.append(dict(off=off, keys=keys, bias=b if bias else None, stride=stride, begin=begin, end=end))

    add([0, 4095, 0, 4096, 4097, 1, 0], 0, 32, bias=True, stride=2)
    add([[0, 1, 4095, 4096, 4097, 12289][i % 6] for i in range(16)], 0, 20)
    add([12289], 4, 20)
    add([4097, 0, 12289], 0, 13, bias=True, stride=3)
    add([4096, 4097, 5], 0, 32, gen=lambda m: np.full(m, 77, np.uint64))                        # every pass trivial
    add([12289, 4095], 0, 32, gen=lambda m: rng.randint(0, 2 ** 24, m, dtype=np.uint64) << 8)    # only the first
    add([1], 0, 32)
    return cases


def b7_digits(c, i, keys):
    b = 0 if c["bias"] is None else int(c["bias"][i])
    nb = 8 * -(-(c["end"] - c["begin"]) // 8)
    k = (keys.astype(np.uint64) - np.uint64(b)) % np.uint64(2 ** 32)
    return ((k >> np.uint64(c["begin"])) & np.uint64((1 << nb) - 1)).astype(np.uint64)


def b7_oracle(c):
    keys, off = c["keys"], c["off"]
    out_k, out_v = keys.copy(), np.arange(keys.size, dtype=np.uint32)
    for i in range(len(off) - 1):
        a, e = off[i], off[i + 1]
        o = np.argsort(b7_digits(c, i, keys[a:e]), kind="stable")
        out_k[a:e], out_v[a:e] = keys[a:e][o], (a + o).astype(np.uint32)
    return out_k, out_v


# ---------------------------------------------------------------------------------------------------------------------
# running and checking
# ---------------------------------------------------------------------------------------------------------------------
def views_of(sts):
    v = np.zeros((len(sts), 40), f32)
    for i, st in enumerate(sts):
        v[i, :16] = st.viewmatrix.numpy().reshape(16); v[i, 16:32] = st.projmatrix.numpy().reshape(16)
        v[i, 32:35] = st.campos.numpy(); v[i, 35:38] = st.bg.numpy()
        v[i, 38], v[i, 39] = st.tanfovx, st.tanfovy
    return v


def run_bins(cl, sts, tight, lists=True):
    from gs_b200 import rasterizer as R
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a)).cuda()        # noqa: E731
    st = sts[0]
    return R.bin_views(d(views_of(sts)), st.image_height, st.image_width, 0, 1.0, d(cl["means3D"]), d(cl["shs"]),
                       d(cl["opacities"]), d(cl["scales"]), d(cl["rotations"]), tight, lists)


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else x


def check_bins(tag, cl, sts, tight, pres=None):
    """run the step's binning twice, check every view against the oracles; returns the first run"""
    a = run_bins(cl, sts, tight)
    b = run_bins(cl, sts, tight)
    for k in a:
        if isinstance(a[k], list):
            assert all(torch.equal(x, y) for x, y in zip(a[k], b[k])) if not isinstance(a[k][0], int) else a[k] == b[k], k
        elif a[k] is not None:
            assert torch.equal(a[k], b[k]), f"{tag}: {k} differs between two runs"
    N = len(cl["means3D"])
    for v, st in enumerate(sts):
        p = pre(cl, st) if pres is None else pres[v]
        gx, gy = p["grid"]
        t = f"{tag} view {v}"
        radii, tiles = _np(a["radii"][v]), _np(a["tiles_touched"][v])
        assert np.array_equal(radii, p["radii"].numpy()), f"{t}: radii differ from gs_oracle.preprocess"
        ot = p["tiles_touched"].numpy()
        spans = _np(a["spans"][v]).astype(np.uint32) if tight else None
        if tight:
            assert np.all(tiles <= ot) and np.all(tiles[ot == 0] == 0), f"{t}: culled count above the square's"
            whole = spans[:, 0] == SENT
            assert np.array_equal(tiles[whole & (ot > 0)], ot[whole & (ot > 0)]), f"{t}: whole-square count"
            rows = np.stack([(spans[:, r >> 1] >> (16 * (r & 1))) & 0xFFFF for r in range(8)], 1).astype(np.int64)
            vis = (ot > 0) & ~whole
            assert np.array_equal((rows[vis] >> 8).sum(1), tiles[vis]), f"{t}: span counts disagree with tiles_touched"
            w, h = (p["rect_max"] - p["rect_min"]).numpy().T
            assert np.all(((rows[vis] & 255) + (rows[vis] >> 8) <= w[vis, None]) | ((rows[vis] >> 8) == 0))
            assert np.all((rows[vis] >> 8)[np.arange(8)[None, :] >= h[vis, None]] == 0), f"{t}: span past the square"
        else:
            assert np.array_equal(tiles, ot), f"{t}: tiles_touched differs from gs_oracle.preprocess"
        ref = oracle_view(p, spans, tiles.astype(np.int64))
        assert np.array_equal(_np(a["sorted_ids"][v]), ref["order"]), f"{t}: depth order"
        assert np.array_equal(_np(a["sorted_dkeys"][v]), ref["sorted_dkeys"]), f"{t}: sorted depth keys"
        assert np.array_equal(_np(a["offsets"][v]), ref["offsets"]), f"{t}: scan offsets"
        assert a["totals"][v] == ref["total"], f"{t}: total {a['totals'][v]} vs {ref['total']}"
        pl, tk = _np(a["point_list"][v]), _np(a["tile_keys"][v])
        assert not (pl == SENT).any() and not (tk == SENT).any(), f"{t}: a pair slot was never written"
        assert np.all(tk < gx * gy), f"{t}: tile key past the tile count"
        assert np.array_equal(np.bincount(pl, minlength=N)[:N], tiles), f"{t}: pairs per Gaussian != tiles_touched"
        assert np.array_equal(tk, ref["tile_keys"]), f"{t}: tile keys"
        assert np.array_equal(pl, ref["point_list"]), f"{t}: point_list"
        rg = _np(a["ranges"][v])
        assert np.array_equal(rg, ref["ranges"].astype(np.int64)), f"{t}: ranges"
        used = rg[:, 1] > rg[:, 0]
        assert np.all(rg[~used] == 0), f"{t}: an empty tile's range is not [0, 0]"
        order = np.argsort(rg[used, 0])
        s, e = rg[used, 0][order], rg[used, 1][order]
        assert (s.size == 0 and pl.size == 0) or (s[0] == 0 and e[-1] == pl.size and np.array_equal(s[1:], e[:-1]))
    return a


gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# B1 depth sort
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("far", [False, True])
@pytest.mark.parametrize("N", [1, 31, 32, 33, 4095, 4096, 4097, 12289])
def test_b1_depth_sort(N, far):
    cl = b1_cloud(N, far)
    sts = [b1_settings(), b1_settings(away=True)]
    for tight in (False, True):
        a = check_bins(f"B1 N={N} far={far} tight={tight}", cl, sts, tight)
        assert a["totals"][1] == 0 and (_np(a["sorted_dkeys"][1]) == SENT).all()


@gpu
def test_b1_one_visible():
    cl = cloud(33, seed=13)
    cl["means3D"][:, 2] = 3.0                       # behind the camera at z = 1.75
    cl["means3D"][17] = (0, 0, 0)
    a = check_bins("B1 one visible", cl, [settings(64, 64)], True)
    assert (_np(a["radii"][0]) > 0).sum() == 1 and _np(a["sorted_ids"][0])[0] == 17


# ---------------------------------------------------------------------------------------------------------------------
# B2 scan and the per-view pair limit
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("N", B2_SIZES)
def test_b2_scan(N):
    cl = small_cloud(N, seed=N % 1000)
    for tight in ((False, True) if N < 10000 else (True,)):
        check_bins(f"B2 N={N} tight={tight}", cl, [settings(256, 256)], tight)


def full_frame(n):
    cl = small_cloud(n, seed=14, spread=0.05, tz=(1.7, 1.8), scale=3.0)
    return cl


@gpu
def test_b2_pair_limit():
    """one pair past 2^30 - 1 in a view is refused with the library's message, before the pairs are allocated, by the
    step's binning and by the one-view forward; the next call works; exactly 2^30 - 1 pairs bin"""
    from gs_b200 import rasterizer as R
    st = settings(1920, 1080)
    over = full_frame(131587)
    with pytest.raises(RuntimeError, match=r"too many \(tile,splat\) pairs in one view: 1073749920"):
        run_bins(over, [st], True, lists=False)
    rs = lambda s: R.GaussianRasterizationSettings(                          # noqa: E731
        s.image_height, s.image_width, s.tanfovx, s.tanfovy, s.bg.cuda(), 1.0, s.viewmatrix.cuda(),
        s.projmatrix.cuda(), 0, s.campos.cuda(), False, False)
    d = lambda k, c: torch.as_tensor(c[k]).cuda()                            # noqa: E731
    fw = lambda c: R.forward_with_state(rs(st), d("means3D", c), d("opacities", c), shs=d("shs", c),  # noqa: E731
                                        scales=d("scales", c), rotations=d("rotations", c))
    with pytest.raises(RuntimeError, match=r"too many \(tile,splat\) pairs in one view: 1073749920"):
        fw(over)
    check_bins("B2 after refusal", small_cloud(3000), [settings(256, 256)], True)
    one = small_cloud(400, seed=15, scale=1e-4, spread=0.5)
    one = {k: v[pre(one, st)["tiles_touched"].numpy() == 1][:LIMIT_SMALL] for k, v in one.items()}
    at = _concat(full_frame(131586), one)
    p = pre(at, st)
    assert int(p["tiles_touched"].sum()) == 2 ** 30 - 1
    out = fw(at)
    assert out["num_rendered"] == 2 ** 30 - 1
    rg = out["ranges"].long()
    assert int((rg[:, 1] - rg[:, 0]).sum()) == 2 ** 30 - 1
    del out
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# B3 emit and spans
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("size", [(4096, 128), (272, 144)])
def test_b3_emit_spans(size):
    W, H = size
    cl = b3_cloud(W, H)
    st = settings(W, H)
    p = pre(cl, st)
    for tight in (False, True):
        a = check_bins(f"B3 {W}x{H} tight={tight}", cl, [st], tight, pres=[p])
    # every tile of its square where some pixel centre reaches alpha >= (1 + 2^-18)/255 with power <= 0 is listed
    # (culled lists; beyond the 3-sigma square the package lists nothing either)
    pl, tk = _np(a["point_list"][0]), _np(a["tile_keys"][0])
    gx = p["grid"][0]
    xy = p["xy"].detach().numpy().astype(np.float64)
    con = p["conic"].detach().numpy().astype(np.float64)
    op = cl["opacities"][:, 0].astype(np.float64)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    tx_of, ty_of = xs.astype(np.int64) // 16, ys.astype(np.int64) // 16
    tile_of = ty_of * gx + tx_of
    rmin, rmax = p["rect_min"].numpy(), p["rect_max"].numpy()
    checked = 0
    for i in np.nonzero(_np(a["radii"][0]) > 0)[0]:
        dx, dy = xy[i, 0] - xs, xy[i, 1] - ys
        power = -0.5 * (con[i, 0] * dx * dx + con[i, 2] * dy * dy) - con[i, 1] * dx * dy
        hit = (power <= 0) & (op[i] * np.exp(np.minimum(power, 0)) >= (1 + 2 ** -18) / 255)
        hit &= (tx_of >= rmin[i, 0]) & (tx_of < rmax[i, 0]) & (ty_of >= rmin[i, 1]) & (ty_of < rmax[i, 1])
        need = np.unique(tile_of[hit])
        listed = np.unique(tk[pl == i])
        missing = np.setdiff1d(need, listed)
        assert missing.size == 0, f"B3 {W}x{H}: Gaussian {i} reaches 1/255 in unlisted tiles {missing[:8]}"
        checked += need.size > 0
    assert checked > 10


# ---------------------------------------------------------------------------------------------------------------------
# B4 tile sort and ranges
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("size", B4_SIZES)
def test_b4_tile_sort(size):
    W, H = size
    cl = cloud(3000, seed=16, scale=0.02)
    for tight in (False, True):
        check_bins(f"B4 {W}x{H} tight={tight}", cl, [settings(W, H)], tight)


# ---------------------------------------------------------------------------------------------------------------------
# B5 the step's chunks
# ---------------------------------------------------------------------------------------------------------------------
B5_EMPTY = {1: [], 2: [0], 16: [0, 7, 15], 17: [0, 4, 8, 9, 16], 33: [0, 10, 11, 21, 32]}


@gpu
@pytest.mark.parametrize("V,N", [(1, 4097), (2, 4097), (16, 4097), (17, 4095), (17, 4096), (17, 4097), (33, 4097)])
def test_b5_chunks(V, N):
    """empty views first, middle and last in a chunk (17 views run as 9 + 8, 33 as 11 + 11 + 11); near and far views
    whose pair counts differ more than 10 times"""
    cl = cloud(N, seed=17, scale=0.2)
    sts = [settings(96, 80, away=True) if v in B5_EMPTY[V] else
           settings(96, 80, radius=(0.9 if v % 2 else 30.0), azim=23.0 * v, elev=7.0 * (v % 5)) for v in range(V)]
    a = check_bins(f"B5 V={V} N={N}", cl, sts, True)
    tot = a["totals"]
    assert all(tot[v] == 0 for v in B5_EMPTY[V])
    live = [t for v, t in enumerate(tot) if v not in B5_EMPTY[V]]
    if len(live) > 1:
        assert max(live) > 10 * min(live)


# ---------------------------------------------------------------------------------------------------------------------
# B6 non-finite and degenerate covariances
# ---------------------------------------------------------------------------------------------------------------------
def _render_views(cl, sts):
    from gs_b200 import _lib
    from gs_b200 import rasterizer as R
    d = lambda a: torch.as_tensor(np.ascontiguousarray(a)).cuda()        # noqa: E731
    vh = views_of(sts)
    V, H, W = len(sts), sts[0].image_height, sts[0].image_width
    img = torch.empty(V, 5, H, W, device="cuda")
    ins = [d(cl[k]) for k in ("means3D", "shs", "opacities", "scales", "rotations")]
    pairs = C.c_int64(0)
    vd = d(vh)
    _lib.check(_lib.lib.gs_b200_render_views(V, H, W, 0, 1.0, C.c_void_p(vh.ctypes.data), C.c_void_p(vd.data_ptr()),
                                             len(cl["means3D"]), 1, C.c_void_p(ins[0].data_ptr()),
                                             C.c_void_p(ins[1].data_ptr()), None, C.c_void_p(ins[2].data_ptr()),
                                             C.c_void_p(ins[3].data_ptr()), C.c_void_p(ins[4].data_ptr()),
                                             C.c_void_p(img.data_ptr()), None, C.byref(pairs), R._stream()))
    torch.cuda.synchronize()
    return img.cpu()


def _raster(cl, st, mode):
    """one-view forward + backward through GaussianRasterizer at tile-culling mode `mode`"""
    from gs_b200 import rasterizer as R
    prev = R.get_tile_culling()
    R.set_tile_culling(mode)
    try:
        rs = R.GaussianRasterizationSettings(st.image_height, st.image_width, st.tanfovx, st.tanfovy, st.bg.cuda(), 1.0,
                                             st.viewmatrix.cuda(), st.projmatrix.cuda(), 0, st.campos.cuda(), False,
                                             False)
        keys = [k for k in ("means3D", "shs", "opacities", "scales", "rotations", "cov3D_precomp") if k in cl]
        inp = {k: torch.as_tensor(cl[k]).cuda().requires_grad_(True) for k in keys}
        m2 = torch.zeros(len(cl["means3D"]), 3, device="cuda", requires_grad=True)
        color, radii, depth, alpha = R.GaussianRasterizer(rs)(
            means3D=inp["means3D"], means2D=m2, opacities=inp["opacities"], shs=inp["shs"],
            scales=inp.get("scales"), rotations=inp.get("rotations"), cov3D_precomp=inp.get("cov3D_precomp"))
        g = torch.Generator(device="cuda").manual_seed(0)
        up = torch.rand(5, st.image_height, st.image_width, device="cuda", generator=g) - 0.5
        ((color * up[:3]).sum() + (depth * up[3:4]).sum() + (alpha * up[4:]).sum()).backward()
        torch.cuda.synchronize()
        grads = {k: v.grad.cpu() for k, v in inp.items()}
        grads["means2D"] = m2.grad.cpu()
        return torch.cat([color, depth, alpha]).detach().cpu(), radii.cpu(), grads
    finally:
        R.set_tile_culling(prev)


@gpu
def test_b6_nonfinite_extent():
    """NaN extents are culled (radius 0, no tile, no depth key) and infinite ones saturate to a full-screen square, in
    the step's binning and the one-view path, culled and not; the image equals the image of the scene without the bad
    Gaussians bit for bit, and every other Gaussian's gradient is unchanged"""
    cl = b6_cloud()
    good = {k: v[:64] for k, v in cl.items()}
    sts = [settings(128, 96, azim=30.0, elev=20.0), settings(128, 96), settings(128, 96, azim=-50.0, elev=-10.0)]
    for tight in (False, True):
        a = check_bins(f"B6 tight={tight}", cl, sts, tight)
        r = _np(a["radii"])
        assert (r[:, B6_BAD] == 0).any() and (r[:, B6_BAD] == 2 ** 31 - 1).any()
    assert torch.equal(_render_views(cl, sts), _render_views(good, sts)), "B6: bad Gaussians change the step's images"
    for mode in (0, 2):
        for st in sts:
            img, radii, g = _raster(cl, st, mode)
            img0, _, g0 = _raster(good, st, mode)
            assert np.array_equal(radii.numpy(), pre(cl, st)["radii"].numpy())
            assert torch.equal(img, img0), f"B6 mode {mode}: bad Gaussians change the image"
            for k in g0:
                assert torch.equal(g[k][:64], g0[k]), f"B6 mode {mode}: {k} gradient of the good Gaussians changed"


@gpu
def test_b6_precomputed_covariance():
    """a negative-definite cov3D_precomp is culled, an indefinite one binned as the oracle bins it; the image without
    the culled one is unchanged"""
    from gs_b200 import rasterizer as R
    cl = b6_cov_cloud()
    st = settings(128, 96, azim=30.0, elev=20.0)
    p = pre(cl, st)
    d = lambda k: torch.as_tensor(cl[k]).cuda()                              # noqa: E731
    rs = R.GaussianRasterizationSettings(96, 128, st.tanfovx, st.tanfovy, st.bg.cuda(), 1.0, st.viewmatrix.cuda(),
                                         st.projmatrix.cuda(), 0, st.campos.cuda(), False, False)
    prev = R.get_tile_culling()
    R.set_tile_culling(0)
    try:
        out = R.forward_with_state(rs, d("means3D"), d("opacities"), shs=d("shs"), cov3D_precomp=d("cov3D_precomp"))
    finally:
        R.set_tile_culling(prev)
    assert np.array_equal(out["radii"].cpu().numpy(), p["radii"].numpy())
    assert p["radii"][64] == 0 and p["radii"][65] > 0
    ref = oracle_view(p, None)
    assert np.array_equal(out["point_list"].cpu().numpy().astype(np.int64), ref["point_list"].astype(np.int64))
    assert np.array_equal(out["ranges"].cpu().numpy().astype(np.int64), ref["ranges"].astype(np.int64))
    drop = {k: np.delete(v, 64, axis=0) for k, v in cl.items()}
    for mode in (0, 2):
        img, _, _ = _raster(cl, st, mode)
        img0, _, _ = _raster(drop, st, mode)
        assert torch.equal(img, img0)


# ---------------------------------------------------------------------------------------------------------------------
# B7 the segmented sort, direct
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("case", range(len(b7_cases())))
def test_b7_segmented_sort(case):
    from gs_b200 import rasterizer as R
    c = b7_cases()[case]
    keys = torch.as_tensor(c["keys"].view(np.int32).copy()).cuda()
    vals = torch.arange(keys.numel(), dtype=torch.int32, device="cuda")
    bias = None
    if c["bias"] is not None:
        b = np.full(len(c["bias"]) * c["stride"], 0x5A5A5A5A, np.uint32)
        b[::c["stride"]] = c["bias"]
        bias = torch.as_tensor(b.view(np.int32)).cuda()
    rk, rv = b7_oracle(c)
    runs = [R.sort_pairs_segmented(keys, vals, c["off"], c["begin"], c["end"], bias, c["stride"]) for _ in range(2)]
    for k, v in runs:
        assert np.array_equal(k.cpu().numpy().view(np.uint32), rk), f"B7 case {case}: keys"
        assert np.array_equal(v.cpu().numpy().view(np.uint32), rv), f"B7 case {case}: values (stability)"
