"""CPU premises of the optimisation-step edge scenes in `test_gpu_optim_edges.py`: each scene's inputs really reach the
edge it is there for (saturations, the normalize clamp, the scalar SH path, subnormal squares, rule boundaries, pyramid
parities, a negative mean cs), and the float64 loss reference runs."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import test_gpu_optim_edges as E

CPU = torch.device("cpu")


def _norm32(q):
    """fp32 sum of squares in order, then sqrt (what any fp32 evaluation gives on these rows)"""
    q = q.numpy().astype(np.float32)
    s = np.float32(0)
    for v in q:
        s = np.float32(s + np.float32(v * v))
    return float(np.sqrt(s, dtype=np.float32))


def test_s1_premise():
    ro, rs, rr = E.s1_inputs()
    o = torch.sigmoid(ro)
    assert bool((o == 0).any()) and bool((o == 1).any())                     # both fp32 saturations
    assert float(ro.min()) == -104.0 and float(ro.max()) == 104.0
    e64 = torch.exp(rs.double())
    assert bool((e64 > E.FLT_MAX).any()) and bool(((e64 > 3.39e38) & (e64 <= E.FLT_MAX)).any())
    q = E.quaternion_rows()
    n64 = q.double().norm(dim=1)
    assert float(n64[0]) == 0.0 and float(n64[1]) < 1e-12 and 0.8e-12 < float(n64[2]) < 1e-12
    assert float(n64[3]) > 1e-12 and _norm32(q[3]) == float(np.float32(1e-12))  # strict clamp: exactly 1e-12f, not clamped
    assert abs(float(n64[4]) - 1) < 1e-6 and abs(float(n64[5]) / 1e18 - 1) < 1e-6
    assert torch.equal(rr[-6:], q)


def test_s2_premise():
    for N in (4096, 4097, 4098, 4099):
        # the SH block starts 3N floats into the packed buffers: 16-byte aligned (128-bit kernel) only for N % 4 == 0
        assert ((3 * N * 4) % 16 == 0) == (N % 4 == 0)
    assert [3 * M % 4 != 0 for M in (1, 4, 9, 16)] == [True, False, True, False]   # float4s straddle rows at M = 1, 9
    N, M = 4097, 4
    raw, gact = E.s2_inputs(N, M, 0)
    xyz, shs, op, sc, ro = E.split(raw, N, M)
    assert bool((torch.sigmoid(op) == 1).any()) and bool((torch.sigmoid(op) == 0).any())
    # gradients whose (1 - b2) g^2 is subnormal or flushes in fp32, and the largest 1e2
    a = gact.abs()
    sq = (1 - E.B2) * a.double() ** 2
    assert bool(((sq > 0) & (sq < 2.0 ** -126)).any()) and float(a.max()) > 100 and bool((a == 0).any())
    # rotation rows where g is nearly parallel to r: the projection cancels
    gr = E.split(gact, N, M)[4]
    par = slice(6, 6 + E.N_PAR)
    cos = (F.normalize(ro[par].double(), dim=1) * F.normalize(gr[par].double(), dim=1)).sum(1).abs()
    assert float(cos.min()) > 0.999
    # below F.normalize's clamp the reference gradient is plain g / 1e-12: the projection formula differs there
    G = E.chain64(raw, gact, 1.0, N, M)
    Gr = E.split(G, N, M)[4]
    assert torch.allclose(Gr[1], gr[1].double() / 1e-12, rtol=1e-12) and torch.allclose(Gr[2], gr[2].double() / 1e-12, rtol=1e-12)
    r, g = ro[2].double(), gr[2].double()
    proj = (g - r * (r @ g) / (r @ r)) / 1e-12
    assert float((proj - Gr[2]).norm() / Gr[2].norm()) > 0.01
    # the all-zero rows, and the history of later steps is nonzero elsewhere
    for t in E.split(gact, N, M):
        assert bool((t[N - E.N_ZERO:] == 0).all())
    m, v = E.history(G, 1000, 0, N, M)
    assert bool((v > 0).any()) and bool((m[: 3 * N] != 0).any()) and bool((E.split(v, N, M)[0][N - E.N_ZERO:] == 0).all())
    assert len(set(E.LRS.tolist())) == 6


def test_s3_premise():
    calls = E.s3_calls()
    assert len(calls) == 5
    r = torch.cat([c[1] for c in calls])
    assert set(r.tolist()) == set(E.S3_RADII)
    gm = torch.cat([c[0][:, :2] for c in calls]).abs()
    sq = gm * gm                                                                       # fp32 squares
    assert bool(((gm > 0) & (sq == 0)).any())                                          # squares that flush to zero
    assert bool(((gm > 0) & (sq > 0) & (sq < 2.0 ** -126)).any())                       # subnormal squares
    assert bool(torch.isinf(sq).any()) and float(gm.max()) >= 1e30                      # squares that overflow


def test_s4_premise():
    b, percent_dense, min_op = E.s4_boundaries(CPU)
    for k in ("pd", "big", "op"):
        eq, up, dn = b[k]
        assert eq and up != eq[0] and dn != eq[0], k
    # the children's exp(log(s / 1.6)) skips values: the inputs nearest the threshold from either side stand for it
    _, up, dn = b["child"]
    c = torch.exp(torch.log(torch.exp(torch.tensor([up, dn])) / 1.6))
    assert float(c[0]) > 0.4 > float(c[1]) and float(c[0] - c[1]) < 1e-6
    assert abs(percent_dense - 0.01) < 1e-6 and abs(min_op - 0.005) < 1e-6
    assert float(torch.exp(torch.tensor([b["big"][0][0]]))[0]) == float(np.float32(0.1) * np.float32(E.EXTENT))
    N, M = 257, 16
    st = E.s4_state(N, M, CPU)
    g = st["acc"] / st["den"]
    assert bool((g == np.float32(E.MAX_GRAD)).any()) and bool(g.isnan().any()) and bool(g.isinf().any())
    sc = E.split(st["raw"], N, M)[3]
    scal = torch.exp(sc).max(1).values
    assert bool((scal == percent_dense * E.EXTENT).any()) and bool((scal == np.float32(0.4)).any())
    op = E.split(st["raw"], N, M)[2][:, 0]
    assert bool((torch.sigmoid(op) == min_op).any())
    # split parents whose children are pruned: the z row differs from the rank among the kept ones
    idx_s = E.split_parents(st, N, M, CPU)
    child_bad = (torch.sigmoid(op[idx_s]) < min_op) | (torch.exp(torch.log(torch.exp(sc[idx_s]) / 1.6)).max(1).values > 0.4)
    assert 0 < int(child_bad.sum()) < idx_s.numel() and not bool(child_bad[-1])


def test_s5_premise():
    from gs_b200 import losses
    # the float64 reference runs (the window follows the input's dtype)
    img, ref, mask = E.s5_inputs("random", 163, 322)
    v = losses.ms_ssim(ref[None].double(), img[None, :3].clamp(0, 1).double())
    assert v.dtype == torch.float64
    l64, g64 = E.loss_ref(img, ref, mask, 0.2, 3.0, 1.0, torch.float64)
    assert g64.dtype == torch.float64 and bool(torch.isfinite(g64).all())

    def pyr(n):
        out = [n]
        for _ in range(4):
            n = (n + (n & 1)) // 2
            out.append(n)
        return out
    assert pyr(1080) == [1080, 540, 270, 135, 68] and pyr(1920) == [1920, 960, 480, 240, 120]   # H odd at level 3, W even
    assert pyr(161)[-1] - 10 == 1 and pyr(163)[0] % 2 == 1                                     # a single valid SSIM row
    # exact 0 and 1 and one ulp outside, with a nonzero L1 gradient there
    img, ref, _ = E.s5_inputs("clamp", 163, 322)
    for v in (0.0, 1.0, E.f32_next(0.0, -1), E.f32_next(1.0, 1)):
        assert bool((img[:3] == v).any()), v
    # the anti-correlated channel drives a level's mean cs below zero
    img, ref, mask = E.s5_inputs("anticorr", 163, 322)
    X, Y = (ref * mask)[None].double(), (img[:3].clamp(0, 1) * mask)[None].double()
    win = losses._gauss_1d(dtype=torch.float64)
    neg = False
    for _ in range(4):
        _, cs = losses._ssim_cs(X, Y, win)
        neg |= bool(cs[0, 0] < 0)
        pad = [s % 2 for s in X.shape[2:]]
        X, Y = F.avg_pool2d(X, 2, padding=pad), F.avg_pool2d(Y, 2, padding=pad)
    assert neg
    assert math.isfinite(float(l64))
