"""Optimisation-step kernels around the rasterizer against a float64 evaluation of the same operation, at the shapes and
edges training takes: the activation at sigmoid / exp saturation and at F.normalize's clamp (S1), the fused chain rule
+ Adam on the vector and the scalar SH path, with data-parallel gradient scales, late steps and gradients from 0 to
1e2 (S2), the densification statistics (S3), densify plan + apply at every rule boundary and in the structural corner
cases (S4), and the image loss up to 1080p (S5).  Every scene has a CPU test of its premise
(`test_optim_edges_cpu.py`).

References.  Activation: torch.sigmoid / exp / F.normalize in float64 on the fp32 inputs.  Chain rule + Adam:
torch.optim.Adam(eps=1e-15) itself (the reference's optimiser) over float64 leaf tensors, with the gradients from
float64 autograd through sigmoid, exp and F.normalize; its state (step, exp_avg, exp_avg_sq) is loaded from the
kernel's fp32 state, so every comparison is one step's error.  Where fp32's sigmoid is exactly 0 or 1 the fp32 chain
rule gradient is exactly 0 while float64 still gives a full lr step; for those rows the reference takes the fp32
autograd gradient (0) and the kernel must agree exactly.  Statistics: float64 from the kernel's previous state, one
call at a time.  Densification: the torch rules of `GaussianTrainer._densify_and_prune_torch` in fp32 on the same
device (decisions, counts, order and every copied row bit for bit) and, for the split children, R(q/|q|)(exp(s) z) +
xyz and log(exp(s)/1.6) in float64 with the same z.  Loss: `gs_b200.losses.training_loss` in float64 with autograd on
the fp32 inputs (on the GPU), the clamp as the trainer applies it.

Per-element bars, u = 2^-24, gamma_n = n u / (1 - n u), TINY = 2^-149 (one subnormal rounding), each times K_ELEM.
CUDA's documented bounds: expf 2 ulp, logf 1 ulp; sqrtf and division are IEEE (no fast-math, csrc/build.sh).
- Activation: sigmoid 1/(1 + expf(-x)): 6u o + TINY, and 1 / FLT_MAX where expf(-x) overflows to inf.  exp: 4u e + TINY (results past FLT_MAX must be inf).
  normalize: gamma_8 |r_k / max(|r|, 1e-12)| + TINY.
- Chain rule (dG, on the |terms|): means / SH 2u |G| (grad_scale's rounding and the product); opacity
  |s g| (o d(1-o) + (1-o) do) + 4u |G| with do = 6u o + TINY; scaling 7u |G|; rotation
  gamma_24 |s| (|g_k| + |r_k| sum_j |r_j g_j| / |r|^2) / |r| + 4 TINY, or 4u |s g_k| / 1e-12 below the clamp.
- Adam, per element from its own terms: e_m = gamma_3 (b1 |m| + (1-b1) |G|) + (1-b1) dG;
  e_v = gamma_4 (b2 v + (1-b2) G^2) + (1-b2)(2 |G| dG + dG^2) + 2 TINY; then through sqrt (min(e_v / 2 sqrt v,
  sqrt e_v) + u sqrt v), / c2 and + eps (2u), m / d (u) and p - st q (2u on st q, u on p).  A tensor-wide bar is
  meaningless here: with eps = 1e-15 every nonzero gradient becomes a step of about lr.
- Statistics: accum + |g| has two roundings: gamma_2 (accum + |g|) + TINY.  denom and max_radii2D exact.
- Children: scaling 6u + 2u |log| ; xyz gamma_5 (sum_j |R_kj e_j| + |xyz_k|) + 30u sum_j |e_j|.
- Loss: no useful worst-case bound through MS-SSIM's products and quotients, so the same restatement in fp32 (cuDNN
  without TF32) sizes the part fp32 cannot avoid: K_LOSS times its largest error per plane; the value adds
  gamma_10 |l| for the kernel's sums (256-term fp32 block trees, then fp64 reds).  Where
  |ref - clamp(img)| is within 4u of its terms the L1 sign is a rounding decision: 2 k1 is allowed there.
Fixed bars, each ten or more times tighter than `test_gpu_trainer.py`'s: activation ACT_REL norm-relative (suite 1e-6
absolute); Adam, per group, ADAM_REL norm-relative on the parameters and MOM_REL on the moments (suite 2e-5 absolute on
parameters of size ~0.5), over the elements whose chain-rule bound dG is below 1e-5 |G| (near sigmoid saturation, where g is nearly parallel
to r, and where G is subnormal, fp32 keeps fewer bits; the per-element bar covers those); statistics STATS_REL norm-relative (suite 1e-6 absolute); children CHILD_REL norm-relative (suite 1e-5
relative); loss LOSS_VAL_REL relative (suite 1e-5) and gradients LOSS_GRAD_MAX of max(|largest gradient|,
scale / 3HW) per plane (suite 2e-4 of the largest).  Tests print each comparison's worst error against both bars."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24
TINY = 2.0 ** -149
K_ELEM = 2.0
K_LOSS = 4.0
FLT_MAX = float(np.finfo(np.float32).max)
ACT_REL = 1e-7
ADAM_REL = 1e-6
MOM_REL = 1e-5
STATS_REL = 1e-7
CHILD_REL = 1e-6
LOSS_VAL_REL = 1e-6
LOSS_GRAD_MAX = 2e-5
B1, B2, EPS = 0.9, 0.999, 1e-15
LRS = np.array([1.6e-3, 2.5e-3, 1.25e-4, 0.05, 0.005, 0.001], dtype=np.float32)      # six distinct group rates
GROUPS = ("xyz", "shs", "opacity", "scaling", "rotation")


def gam(n):
    return n * U / (1.0 - n * U)


def report(name, err, bar, ref=None):
    """worst error / element bar, and the norm-relative error; returns (ratio, rel)"""
    err = torch.as_tensor(err, dtype=torch.float64).abs().reshape(-1)
    bar = torch.as_tensor(bar, dtype=torch.float64).reshape(-1).to(err.device)
    ratio = float((err / bar.clamp_min(1e-300)).max()) if err.numel() else 0.0
    rel = float(err.norm() / max(float(torch.as_tensor(ref, dtype=torch.float64).norm()), 1e-300)) if ref is not None else float("nan")
    print(f"{name}: max err {float(err.max()) if err.numel() else 0.0:.3g}, worst err/bar {ratio:.3g}, norm-rel {rel:.3g}")
    return ratio, rel


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def f32_next(x, n=1):
    """x moved n fp32 ulps (n < 0: down)"""
    v = np.float32(x)
    for _ in range(abs(n)):
        v = np.nextafter(v, np.float32(np.inf if n > 0 else -np.inf), dtype=np.float32)
    return float(v)


# ---------------------------------------------------------------------------------------------------------------------
# S1 activation
# ---------------------------------------------------------------------------------------------------------------------
def boundary_quaternion():
    """fp32 components whose fp32 norm rounds to exactly 1e-12f while the exact norm lies above 1e-12 (double): no
    clamp in either precision, so the kernel's clamp test must be strict"""
    return torch.tensor([f32_next(1e-12, 0), 1.2e-16, 0.0, 0.0], dtype=torch.float32)


def quaternion_rows(seed=0):
    """norms 0, 1e-13, just below 1e-12, exactly 1e-12f after rounding, 1 and 1e18, random directions"""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for nrm in (0.0, 1e-13, 0.9e-12, None, 1.0, 1e18):
        if nrm is None:
            rows.append(boundary_quaternion())
            continue
        d = torch.randn(4, generator=g, dtype=torch.float64)
        rows.append((d / d.norm() * nrm).float())
    return torch.stack(rows)


def s1_inputs(seed=0):
    g = torch.Generator().manual_seed(seed)
    n_rand = 3000
    lin = torch.linspace(-104.0, 104.0, 2081)                               # expf overflow .. sigmoid rounds to 1
    log_max = float(np.float32(math.log(FLT_MAX)))
    near = torch.tensor([f32_next(log_max, k) for k in range(-3, 4)] + [88.72, 88.73, 89.0, 100.0, -87.0, -103.0, -104.0])
    opac = torch.cat([torch.randn(n_rand, generator=g) * 3, lin, torch.zeros(near.numel() + 6)])
    N = opac.numel()
    scal = torch.randn(N, 3, generator=g) * 2
    scal[n_rand:n_rand + 2081, 0] = torch.linspace(-104.0, 88.72, 2081)
    scal[n_rand + 2081:n_rand + 2081 + near.numel(), 1] = near              # up to and past the fp32 exp overflow
    rots = torch.randn(N, 4, generator=g)
    rots[-6:] = quaternion_rows(seed)
    return opac.contiguous(), scal.contiguous(), rots.contiguous()


def _exp_bar(ref64):
    return K_ELEM * (4 * U * ref64.abs() + TINY)


def check_exp(name, got, ref64):
    """exp outputs: where the float64 value rounds past FLT_MAX the kernel must give inf; within 4u of it either"""
    over = ref64 > FLT_MAX * (1 + 4 * U)
    gap = (ref64 > FLT_MAX * (1 - 4 * U)) & ~over
    assert bool(torch.isinf(got[over]).all()), name
    fin = ~over & ~(gap & torch.isinf(got))
    return report(name, (got.double() - ref64)[fin], _exp_bar(ref64)[fin], ref64[fin])


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.mark.gpu
def test_s1_activation(dev):
    from gs_b200 import _lib
    ro, rs, rr = (t.to(dev) for t in s1_inputs())
    N = ro.numel()
    o, s, r = torch.empty_like(ro), torch.empty_like(rs), torch.empty_like(rr)
    _lib.check(_lib.lib.gs_b200_activate(N, _ptr(ro), _ptr(rs), _ptr(rr), _ptr(o), _ptr(s), _ptr(r), None))
    torch.cuda.synchronize()
    o64, s64, r64 = torch.sigmoid(ro.double()), torch.exp(rs.double()), F.normalize(rr.double(), dim=-1)
    assert bool((o == 0).any()) and bool((o == 1).any())                    # both saturations reached on the device
    # past expf's overflow (x < -log FLT_MAX) o is 0 where the exact value is below 1 / FLT_MAX
    over = torch.where(-ro.double() > math.log(FLT_MAX), 1.0 / FLT_MAX, 0.0)
    ra, rl = report("S1 sigmoid", o.double() - o64, K_ELEM * (6 * U * o64 + TINY + over), o64)
    assert ra <= 1 and rl <= ACT_REL
    ra, rl = check_exp("S1 exp", s, s64)
    assert ra <= 1 and rl <= ACT_REL
    assert bool(torch.isinf(s).any()) and bool((s[torch.isfinite(s)] > 3.39e38).any())
    bar = K_ELEM * (gam(8) * r64.abs() + TINY)
    ra, rl = report("S1 normalize", r.double() - r64, bar, r64)
    assert ra <= 1 and rl <= ACT_REL
    assert bool((r[-6] == 0).all())                                         # norm 0 stays 0


# ---------------------------------------------------------------------------------------------------------------------
# S2 chain rule + Adam
# ---------------------------------------------------------------------------------------------------------------------
def sizes(N, M):
    return [3 * N, 3 * M * N, N, 3 * N, 4 * N]


def split(buf, N, M):
    out, o = [], 0
    for s, shp in zip(sizes(N, M), [(N, 3), (N, M, 3), (N, 1), (N, 3), (N, 4)]):
        out.append(buf[o:o + s].view(*shp)); o += s
    return out


MAGS = (0.0, 1e-24, 1e-22, 1e-20, 1e-12, 1e-9, 1e-6, 1e-3, 0.1, 1.0, 10.0, 1e2)   # g^2 subnormal for the first few
N_ZERO = 32                                                                       # last rows: g = 0, zero history
N_PAR = 64                                                                        # rows whose rotation g ~ r


def s2_inputs(N, M, seed):
    """packed raw parameters and dL/d(activated) with per-element magnitudes MAGS; rows 0-5 carry S1's quaternions,
    rows 6.. g nearly parallel to r, the first rows raw opacity over [-104, 104]; the last N_ZERO rows zero gradient"""
    g = torch.Generator().manual_seed(seed)
    T = sum(sizes(N, M))
    raw = torch.randn(T, generator=g) * 0.5
    xyz, shs, op, sc, ro = split(raw, N, M)
    k = min(N, 2049)
    op[:k, 0] = torch.linspace(-104.0, 104.0, k)
    sc -= 2.0
    nq = min(N, 6)
    ro[:nq] = quaternion_rows(seed)[:nq]
    mag = torch.tensor(MAGS)[torch.randint(0, len(MAGS), (T,), generator=g)]
    gact = mag * (torch.rand(T, generator=g) + 0.5) * torch.where(torch.rand(T, generator=g) < 0.5, -1.0, 1.0)
    gx, gsh, go, gsc, gr = split(gact, N, M)
    par = slice(6, min(N, 6 + N_PAR))
    rn = ro[par] / ro[par].norm(dim=1, keepdim=True)
    gr[par] = rn * (torch.rand(rn.shape[0], 1, generator=g) * 10) + 1e-5 * torch.randn(rn.shape, generator=g)
    for t in (gx, gsh, go, gsc, gr):
        t[N - min(N, N_ZERO):] = 0.0
    return raw.contiguous(), gact.contiguous()


def chain64(raw, gact, gs, N, M):
    """float64 autograd through sigmoid / exp / F.normalize (the trainer's activations) -> packed dL/draw"""
    leaves = [t.double().clone().requires_grad_(True) for t in split(raw, N, M)]
    xyz, shs, op, sc, ro = leaves
    gx, gsh, go, gsc, gr = [t.double() for t in split(gact, N, M)]
    loss = (xyz * gx).sum() + (shs * gsh).sum() + (torch.sigmoid(op) * go).sum() + (torch.exp(sc) * gsc).sum() + \
        (F.normalize(ro, dim=-1) * gr).sum()
    (loss * gs).backward()
    return torch.cat([t.grad.reshape(-1) for t in leaves])


def chain_bound(raw, gact, gs, N, M):
    """per-element bound dG of the kernel's fp32 chain rule (module docstring)"""
    xyz, shs, op, sc, ro = [t.double() for t in split(raw, N, M)]
    gx, gsh, go, gsc, gr = [t.double().abs() * abs(gs) for t in split(gact, N, M)]
    o = torch.sigmoid(op); om = 1.0 - o
    do = 6 * U * o + TINY
    d_op = go * (o * (do + U * om) + om * do) + 4 * U * go * o * om + TINY
    d_sc = 7 * U * gsc * torch.exp(sc) + TINY
    n = ro.norm(dim=1, keepdim=True)
    clamped = n < 1e-12
    nn_ = n.clamp_min(1e-12)
    d_ro_free = gam(24) * (gr + ro.abs() * (ro.abs() * gr).sum(1, keepdim=True) / nn_ ** 2) / nn_ + 4 * TINY
    d_ro = torch.where(clamped, 4 * U * gr / 1e-12 + TINY, d_ro_free)
    return torch.cat([(2 * U * gx + TINY).reshape(-1), (2 * U * gsh + TINY).reshape(-1), d_op.reshape(-1), d_sc.reshape(-1),
                      d_ro.reshape(-1)])


def step_sizes(N, M, step):
    """per element lr / (1 - b1^t), dc / rest following the SH coefficient"""
    bias1 = 1.0 - B1 ** step
    lr = [float(x) / bias1 for x in LRS]
    sh = torch.full((N, M, 3), lr[2], dtype=torch.float64); sh[:, 0] = lr[1]
    return torch.cat([torch.full((3 * N,), lr[0], dtype=torch.float64), sh.reshape(-1), torch.full((N,), lr[3], dtype=torch.float64),
                      torch.full((3 * N,), lr[4], dtype=torch.float64), torch.full((4 * N,), lr[5], dtype=torch.float64)])


def history(G64, step, seed, N, M):
    """a seeded plausible (m, v) before `step`: zero at step 1, else scaled like the gradient; zero on the g = 0 rows"""
    T = G64.numel()
    if step == 1:
        return torch.zeros(T), torch.zeros(T)
    g = torch.Generator().manual_seed(seed + 7)
    sig = G64.abs().cpu() * (torch.rand(T, generator=g, dtype=torch.float64) + 0.5)
    m = ((1 - B1 ** (step - 1)) * sig * torch.randn(T, generator=g, dtype=torch.float64) * 0.5).float()
    v = ((1 - B2 ** (step - 1)) * sig * sig * (torch.rand(T, generator=g, dtype=torch.float64) + 0.5)).float()
    for buf in (m, v):
        for t in split(buf, N, M):
            t[N - min(N, N_ZERO):] = 0.0
    return m, v


def adam_ref64(raw, m0, v0, G, N, M, step):
    """torch.optim.Adam(eps=1e-15) over float64 leaves (six groups: xyz, f_dc, f_rest, opacity, scaling, rotation),
    gradient G, state loaded from the fp32 (m0, v0) before `step`.  Returns packed (p, m, v)."""
    ps, gs_, ms, vs = [split(t.double(), N, M) for t in (raw, G, m0, v0)]
    pick = [lambda t: t[0], lambda t: t[1][:, :1], lambda t: t[1][:, 1:], lambda t: t[2], lambda t: t[3], lambda t: t[4]]
    leaves = []
    for k in range(6):
        leaf = pick[k](ps).clone().requires_grad_(True)
        leaf.grad = pick[k](gs_).clone()
        leaves.append((leaf, pick[k](ms).clone(), pick[k](vs).clone(), float(LRS[k])))
    live = [t for t in leaves if t[0].numel()]                      # M = 1: no f_rest
    opt = torch.optim.Adam([{"params": [leaf], "lr": lr} for leaf, _, _, lr in live], lr=0.0, betas=(B1, B2), eps=EPS)
    for leaf, m, v, _ in live:
        opt.state[leaf] = {"step": torch.tensor(float(step - 1)), "exp_avg": m, "exp_avg_sq": v}
    opt.step()
    out = []
    for what in range(3):
        parts = [leaf.detach() if what == 0 else (m if what == 1 else v) for leaf, m, v, _ in leaves]
        sh = torch.cat([parts[1], parts[2]], dim=1)
        out.append(torch.cat([parts[0].reshape(-1), sh.reshape(-1)] + [t.reshape(-1) for t in parts[3:]]))
    return out


def adam_bounds(G, dG, m0, v0, m_ref, v_ref, p_ref, st, step):
    m0, v0 = m0.double(), v0.double()
    e_m = gam(3) * (B1 * m0.abs() + (1 - B1) * G.abs()) + (1 - B1) * dG + TINY
    e_v = gam(4) * (B2 * v0 + (1 - B2) * G * G) + (1 - B2) * (2 * G.abs() * dG + dG * dG) + 2 * TINY
    s = v_ref.sqrt()
    e_s = torch.minimum(e_v / (2 * s), e_v.sqrt()) + U * s
    c2 = math.sqrt(1.0 - B2 ** step)
    d = s / c2 + EPS
    e_d = (e_s + 2 * U * s) / c2 + U * d + U * EPS
    d_lo = (d - e_d).clamp_min(0.5 * EPS)
    q = m_ref / d
    e_q = e_m / d_lo + m_ref.abs() * e_d / (d * d_lo) + U * q.abs()
    e_p = st * (e_q + 2 * U * q.abs()) + U * p_ref.abs() + TINY
    return e_p, e_m, e_v


def _adam_kernel(raw, m0, v0, gact, N, M, step, gs):
    from gs_b200 import _lib
    p, m, v = raw.clone(), m0.clone(), v0.clone()
    _lib.check(_lib.lib.gs_b200_adam_step(N, M, C.c_void_p(LRS.ctypes.data), B1, B2, EPS, step, gs, _ptr(gact), _ptr(p), _ptr(m),
                                          _ptr(v), None))
    torch.cuda.synchronize()
    return p, m, v


def _group_slices(N, M):
    o, out = 0, {}
    for name, s in zip(GROUPS, sizes(N, M)):
        out[name] = slice(o, o + s); o += s
    return out


S2_STEPS = (1, 2, 10, 1000, 30000)
S2_SCALES = (1.0, 0.5, 1.0 / 3.0)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 4, 9, 16])
@pytest.mark.parametrize("N", [4096, 4097, 4098, 4099])
def test_s2_chain_rule_adam(dev, N, M):
    """N % 4 == 0 runs the SH block through the 128-bit kernel, the others through the scalar kernel; M = 1 and 9 make a
    float4 straddle two rows.  Each (step, grad_scale) is one step from a seeded history, checked group by group."""
    gsl = _group_slices(N, M)
    worst = {k: [0.0] * 6 for k in GROUPS}
    for si, step in enumerate(S2_STEPS):
        for gi, gs in enumerate(S2_SCALES):
            seed = 1000 * N + 10 * M + 3 * si + gi
            raw, gact = (t.to(dev) for t in s2_inputs(N, M, seed))
            G = chain64(raw, gact, gs, N, M)
            dG = chain_bound(raw, gact, gs, N, M)
            # fp32's sigmoid at 0 or 1: the fp32 chain-rule gradient is exactly 0 (the reference takes it from fp32)
            op = split(raw, N, M)[2].reshape(-1)
            o32 = torch.sigmoid(op)
            sat = (o32 == 0) | (o32 == 1)
            G[gsl["opacity"]] = torch.where(sat, torch.zeros_like(op, dtype=torch.float64), G[gsl["opacity"]])
            dG[gsl["opacity"]] = torch.where(sat, torch.zeros_like(op, dtype=torch.float64), dG[gsl["opacity"]])
            m0, v0 = (t.to(dev) for t in history(G, step, seed, N, M))
            p, m, v = _adam_kernel(raw, m0, v0, gact, N, M, step, gs)
            p_ref, m_ref, v_ref = adam_ref64(raw, m0, v0, G, N, M, step)
            st = step_sizes(N, M, step).to(dev)
            e_p, e_m, e_v = adam_bounds(G, dG, m0, v0, m_ref, v_ref, p_ref, st, step)
            well = (dG <= 1e-5 * G.abs()) | (G == 0)       # fixed bars: where fp32's chain rule keeps 16 bits
            for name, sl in gsl.items():
                for j, (got, ref, bar, lim) in enumerate(((p, p_ref, e_p, ADAM_REL), (m, m_ref, e_m, MOM_REL), (v, v_ref, e_v, MOM_REL))):
                    err = (got[sl].double() - ref[sl]).abs()
                    ratio = float((err / (K_ELEM * bar[sl])).max())
                    w = well[sl]
                    rel = float(err[w].norm() / ref[sl][w].norm().clamp_min(1e-300))
                    assert ratio <= 1.0 and rel <= lim, (name, "pmv"[j], step, gs, ratio, rel)
                    worst[name][j] = max(worst[name][j], ratio)
                    worst[name][3 + j] = max(worst[name][3 + j], rel / lim)
            # g = 0 with a zero history: p, m and v are bit-unchanged
            for name, sl in gsl.items():
                rows = split(torch.arange(sum(sizes(N, M)), device=dev), N, M)[GROUPS.index(name)][N - N_ZERO:].reshape(-1)
                assert torch.equal(p[rows], raw[rows]) and bool((m[rows] == 0).all()) and bool((v[rows] == 0).all()), name
            if step == 1:       # zero history: m = (1 - b1) g, so the kernel's zero / nonzero gradient is visible in m
                mo = m[gsl["opacity"]]
                assert torch.equal(mo[sat] == 0, torch.ones_like(mo[sat], dtype=torch.bool)), "saturated opacity moved"
                assert bool((mo[~sat & (gact[gsl["opacity"]] != 0) & (G[gsl["opacity"]].abs() > 1e-30)] != 0).all())
    for name in GROUPS:
        w = worst[name]
        print(f"S2 N={N} M={M} {name}: worst err/bar p {w[0]:.3g}, m {w[1]:.3g}, v {w[2]:.3g}; "
              f"norm-rel / fixed bar p {w[3]:.3g}, m {w[4]:.3g}, v {w[5]:.3g}")


@pytest.mark.gpu
def test_s2_adam_refuses_step_below_one(dev):
    """step < 1 would make the bias correction 1 - b1^0 = 0"""
    from gs_b200 import _lib
    raw, gact = (t.to(dev) for t in s2_inputs(64, 1, 0))
    m, v = torch.zeros_like(raw), torch.zeros_like(raw)
    before = raw.clone()
    for step in (0, -1):
        with pytest.raises(RuntimeError, match="adam_step"):
            _lib.check(_lib.lib.gs_b200_adam_step(64, 1, C.c_void_p(LRS.ctypes.data), B1, B2, EPS, step, 1.0, _ptr(gact), _ptr(raw),
                                                  _ptr(m), _ptr(v), None))
    torch.cuda.synchronize()
    assert torch.equal(raw, before)


# ---------------------------------------------------------------------------------------------------------------------
# S3 densification statistics
# ---------------------------------------------------------------------------------------------------------------------
S3_N = 4099
S3_RADII = (-1, 0, 1, 2 ** 30)
S3_MAGS = (0.0, 1e-30, 1e-23, 1e-21, 1e-3, 1.0, 1e19, 1e30)


def s3_calls(seed=0, calls=5):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(calls):
        r = torch.tensor(S3_RADII, dtype=torch.int32)[torch.randint(0, 4, (S3_N,), generator=g)]
        mag = torch.tensor(S3_MAGS)[torch.randint(0, len(S3_MAGS), (S3_N, 3), generator=g)]
        gm = (mag * (torch.rand(S3_N, 3, generator=g) + 0.5) * torch.where(torch.rand(S3_N, 3, generator=g) < 0.5, -1.0, 1.0)).float()
        gm[:, 2] = 1e30                                             # the third component is not part of the norm
        out.append((gm.contiguous(), r.contiguous()))
    return out


@pytest.mark.gpu
def test_s3_densify_stats(dev):
    from gs_b200 import _lib
    acc = torch.zeros(S3_N, device=dev); den = torch.zeros(S3_N, device=dev); mr = torch.zeros(S3_N, device=dev)
    worst = (0.0, 0.0)
    for gm, r in s3_calls():
        gm, r = gm.to(dev), r.to(dev)
        a0, d0, m0 = acc.double(), den.clone(), mr.clone()
        _lib.check(_lib.lib.gs_b200_densify_stats(S3_N, _ptr(gm), _ptr(r), _ptr(acc), _ptr(den), _ptr(mr), None))
        torch.cuda.synchronize()
        vis = r > 0
        nrm = gm[:, :2].double().norm(dim=1)
        ref = torch.where(vis, a0 + nrm, a0)
        bar = K_ELEM * (gam(2) * (a0 + nrm) + TINY)
        ra, rl = report("S3 accum", acc.double() - ref, torch.where(vis, bar, torch.full_like(bar, TINY)), ref)
        worst = (max(worst[0], ra), max(worst[1], rl))
        assert ra <= 1 and rl <= STATS_REL
        assert torch.equal(den, torch.where(vis, d0 + 1, d0))
        assert torch.equal(mr, torch.where(vis, torch.maximum(m0, r.float()), m0))
    assert float(mr.max()) == 2.0 ** 30 and bool(torch.isfinite(acc).all())


# ---------------------------------------------------------------------------------------------------------------------
# S4 densify plan + apply
# ---------------------------------------------------------------------------------------------------------------------
MAX_GRAD = 2e-4
EXTENT = 4.0


def _search(dev, centre, fn, target, span=400):
    """fp32 inputs around `centre` whose fn (evaluated on `dev`) equals target exactly, and the nearest inputs whose
    value lies just above and just below it"""
    c = np.float32(centre)
    xs = [c]
    lo = hi = c
    for _ in range(span):
        lo = np.nextafter(lo, np.float32(-np.inf), dtype=np.float32); hi = np.nextafter(hi, np.float32(np.inf), dtype=np.float32)
        xs += [lo, hi]
    x = torch.tensor(np.array(sorted(xs), dtype=np.float32), device=dev)
    y = fn(x)
    t = torch.tensor(np.float32(target), device=dev)
    eq = x[y == t]
    above = x[y > t]; below = x[y < t]
    inc = bool(y[-1] > y[0])
    up = above[0] if inc else above[-1]
    dn = below[-1] if inc else below[0]
    return [float(v) for v in eq], float(up), float(dn)


def s4_boundaries(dev):
    """the rule thresholds and fp32 raw inputs that land on them, evaluated with the device's own expf / logf:
    scal > percent_dense * extent (percent_dense chosen so that the threshold is an attainable exp value),
    scal > 0.1 * extent, the children's exp(log(s / 1.6)) > 0.1 * extent (a chain of roundings that may skip the
    threshold itself: then the nearest inputs either side), sigmoid(op) < min_opacity (min_opacity chosen attainable
    likewise); g >= max_grad is placed directly.  Returns ({rule: (inputs on it, nearest above, nearest below)},
    percent_dense, min_opacity)."""
    dev = torch.device(dev)
    s_pd = float(np.float32(math.log(0.04)))
    thr_pd = float(torch.exp(torch.tensor([s_pd], device=dev))[0])
    percent_dense = thr_pd / EXTENT
    x_op = float(np.float32(math.log(0.005 / 0.995)))
    min_op = float(torch.sigmoid(torch.tensor([x_op], device=dev))[0])
    big = np.float32(0.1) * np.float32(EXTENT)
    b = {}
    b["pd"] = _search(dev, s_pd, torch.exp, thr_pd, 8)
    b["big"] = _search(dev, math.log(0.4), torch.exp, big)
    b["child"] = _search(dev, math.log(0.64), lambda x: torch.exp(torch.log(torch.exp(x) / 1.6)), big)
    b["op"] = _search(dev, x_op, torch.sigmoid, min_op, 8)
    return b, percent_dense, min_op


def s4_state(N, M, dev, seed=0, cap=None):
    """raw (packed), m1, m2, accum, denom with rows cycling through every combination of a gradient choice (at
    max_grad, one ulp either side, 0 / 0, x / 0, random), a scaling choice (on each scaling threshold and the fp32
    inputs either side, random) and an opacity choice (on min_opacity, either side, random); rows past 240 draw a
    combination at random.  cap: trainer capacity (default N)."""
    b, percent_dense, min_op = s4_boundaries(dev)
    g = torch.Generator().manual_seed(seed + N + M)
    T = sum(sizes(N, M))
    raw = torch.randn(T, generator=g) * 0.5
    m1 = torch.randn(T, generator=g) * 1e-3
    m2 = torch.rand(T, generator=g) * 1e-6
    xyz, shs, op, sc, ro = split(raw, N, M)
    mg = np.float32(MAX_GRAD)
    nan = float("nan")
    first = lambda k: b[k][0][0] if b[k][0] else nan
    g_vals = torch.tensor([float(mg), f32_next(mg, 1), f32_next(mg, -1), 0.0, 1e-3, nan])
    d_vals = torch.tensor([1.0, 1.0, 1.0, 0.0, 0.0, 1.0])
    s_vals = torch.tensor([first("pd"), b["pd"][1], b["pd"][2], first("big"), b["big"][1], b["big"][2], first("child"), b["child"][1],
                           b["child"][2], nan])
    o_vals = torch.tensor([first("op"), b["op"][1], b["op"][2], nan])
    acc = torch.rand(N, generator=g) * 4e-4
    den = torch.ones(N)
    sc.copy_(torch.log(torch.rand(N, 3, generator=g) * 0.08 + 1e-3))
    op.copy_(torch.randn(N, 1, generator=g) * 2)
    c = torch.arange(N)
    c = torch.where(c < 240, c, torch.randint(0, 240, (N,), generator=g))
    gv, dv = g_vals[c % 6], d_vals[c % 6]
    acc = torch.where(gv.isnan(), acc, gv); den = torch.where(gv.isnan(), den, dv)
    sv = s_vals[(c // 6) % 10]
    hit = ~sv.isnan()
    k = c % 3
    sc[hit] = (sv[hit] - 1.0)[:, None].expand(-1, 3).clone()
    sc[hit.nonzero()[:, 0], k[hit]] = sv[hit]
    ov = o_vals[(c // 60) % 4]
    op[:, 0] = torch.where(ov.isnan(), op[:, 0], ov)
    return dict(raw=raw, m1=m1, m2=m2, acc=acc.float(), den=den.float(), percent_dense=percent_dense, min_op=min_op, b=b,
                cap=cap)


def _trainer(st, N, M, dev):
    from gs_b200 import trainer
    tr = trainer.GaussianTrainer.__new__(trainer.GaussianTrainer)
    tr.p = trainer.TrainParams(sh_degree=int(round(math.sqrt(M))) - 1, percent_dense=st["percent_dense"])
    tr.device = torch.device(dev); tr.M = M; tr.step_count = 0
    tr._alloc(N)
    if st["cap"]:
        tr._alloc_grow(st["cap"]); tr._bind(N, zero=True)
    tr.raw.copy_(st["raw"]); tr.m1.copy_(st["m1"]); tr.m2.copy_(st["m2"])
    tr.grad_accum.copy_(st["acc"]); tr.denom.copy_(st["den"])
    return tr


def split_parents(st, N, M, dev):
    """indices of the split parents (in order), by the torch rules in fp32 on the device"""
    raw = st["raw"].to(dev)
    sc = split(raw, N, M)[3]
    grads = st["acc"].to(dev) / st["den"].to(dev)
    grads[grads.isnan()] = 0.0
    scal = torch.exp(sc).max(dim=1).values
    return torch.nonzero((grads >= MAX_GRAD) & (scal > st["percent_dense"] * EXTENT))[:, 0]


def run_s4(st, N, M, dev, monkeypatch):
    """(CUDA trainer, CUDA info, torch trainer, torch info, z, split parent indices)"""
    idx_s = split_parents(st, N, M, dev)
    g = torch.Generator().manual_seed(N + 5)
    z = torch.randn(2 * idx_s.numel(), 3, generator=g).to(dev)
    a = _trainer(st, N, M, dev)
    info_a = a.densify_and_prune(MAX_GRAD, st["min_op"], EXTENT, 1.0, normal_samples=z)
    b = _trainer(st, N, M, dev)
    monkeypatch.setattr(torch, "normal", lambda mean, std, generator=None: z * std + mean)
    info_b = b._densify_and_prune_torch(MAX_GRAD, st["min_op"], EXTENT, 1.0)
    monkeypatch.undo()
    return a, info_a, b, info_b, z, idx_s


def check_s4(st, N, M, dev, monkeypatch):
    a, info_a, b, info_b, z, idx_s = run_s4(st, N, M, dev, monkeypatch)
    torch.cuda.synchronize()
    assert info_a == info_b, (info_a, info_b)
    n = a.N
    assert b.N == n
    # children rows: after the survivors and the kept clones
    raw0 = st["raw"].to(dev)
    sc0 = split(raw0, N, M)[3]
    op0 = split(raw0, N, M)[2][:, 0]
    n_sp = idx_s.numel()
    child_bad = (torch.sigmoid(op0[idx_s]) < st["min_op"]) | (torch.exp(torch.log(torch.exp(sc0[idx_s]) / 1.6)).max(1).values > 0.1 * EXTENT)
    kept = torch.nonzero(~child_bad)[:, 0]                       # rank among ALL split parents = row of z
    n_ck = kept.numel()
    first_child = n - 2 * n_ck
    va, vb = a._views(a.raw, n), b._views(b.raw, n)
    for k in GROUPS:
        if k in ("xyz", "scaling"):
            assert torch.equal(va[k][:first_child], vb[k][:first_child]), k
        else:
            assert torch.equal(va[k], vb[k]), k
    for buf in ("m1", "m2"):
        assert torch.equal(getattr(a, buf), getattr(b, buf)), buf
    n_keep = info_a["n_before"] - info_a["pruned"]
    for buf in (a.m1, a.m2):                                      # new rows start with zero moments
        for k, t in a._views(buf, n).items():
            assert bool((t[n_keep:] == 0).all()), k
    if n_ck:
        par = idx_s[kept]
        xyz0, ro0 = split(raw0, N, M)[0], split(raw0, N, M)[4]
        q = ro0[par].double(); q = q / q.norm(dim=1, keepdim=True)
        r_, x_, y_, z_ = q.unbind(1)
        R = torch.stack([1 - 2 * (y_ * y_ + z_ * z_), 2 * (x_ * y_ - r_ * z_), 2 * (x_ * z_ + r_ * y_), 2 * (x_ * y_ + r_ * z_),
                         1 - 2 * (x_ * x_ + z_ * z_), 2 * (y_ * z_ - r_ * x_), 2 * (x_ * z_ - r_ * y_), 2 * (y_ * z_ + r_ * x_),
                         1 - 2 * (x_ * x_ + y_ * y_)], 1).view(-1, 3, 3)
        s = torch.exp(sc0[par].double())
        for c in range(2):
            e = s * z[c * n_sp + kept].double()
            ref = torch.bmm(R, e[:, :, None])[:, :, 0] + xyz0[par].double()
            bar = K_ELEM * (gam(5) * ((R.abs() * e.abs()[:, None, :]).sum(2) + xyz0[par].double().abs()) + 30 * U * e.abs().sum(1, keepdim=True) + TINY)
            rows = slice(first_child + c * n_ck, first_child + (c + 1) * n_ck)
            ra, rl = report(f"S4 N={N} M={M} child {c} xyz", va["xyz"][rows].double() - ref, bar, ref - xyz0[par].double())
            assert ra <= 1 and rl <= CHILD_REL
            ref_s = torch.log(s / 1.6)
            ra, rl = report(f"S4 N={N} M={M} child {c} scaling", va["scaling"][rows].double() - ref_s,
                            K_ELEM * (6 * U + 2 * U * ref_s.abs() + TINY), ref_s)
            assert ra <= 1 and rl <= CHILD_REL
    return info_a, n_sp, n_ck


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 16])
@pytest.mark.parametrize("N", [1, 7, 255, 256, 257, 100_003])
def test_s4_densify_rule_boundaries(dev, N, M, monkeypatch):
    st = s4_state(N, M, dev)
    if N >= 240:        # every boundary really sits on its threshold on this device
        b = st["b"]
        assert b["pd"][0] and b["big"][0] and b["op"][0], b
        print("S4 children's threshold attained exactly on this device:", bool(b["child"][0]))
    info, n_sp, n_ck = check_s4(st, N, M, dev, monkeypatch)
    print(f"S4 N={N} M={M}: {info}, split parents {n_sp}, with kept children {n_ck}")
    if N >= 240:
        assert info["cloned"] > 0 and n_sp > n_ck > 0 and info["pruned"] > n_sp


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["none", "all_clone", "all_split", "all_pruned", "grow"])
def test_s4_densify_structural_cases(dev, case, monkeypatch):
    N, M = 1000, 16
    st = s4_state(N, M, dev, seed=1, cap=None if case == "grow" else 2 * N + 1)   # "grow": the result outgrows the buffers
    raw = st["raw"]
    _, _, op, sc, _ = split(raw, N, M)
    op.fill_(2.0)
    if case == "none":
        st["acc"].fill_(0.0)
        sc.fill_(math.log(0.01))
    elif case in ("all_clone", "grow"):
        st["acc"].fill_(1.0); st["den"].fill_(1.0)
        sc.fill_(math.log(0.01))
    elif case == "all_split":
        st["acc"].fill_(1.0); st["den"].fill_(1.0)
        sc.fill_(math.log(0.2))
    elif case == "all_pruned":
        st["acc"].fill_(0.0)
        op.fill_(-20.0)
    info, n_sp, n_ck = check_s4(st, N, M, dev, monkeypatch)
    print(f"S4 {case}: {info}")
    want = {"none": (0, 0, 0, N), "all_clone": (N, 0, 0, 2 * N), "grow": (N, 0, 0, 2 * N), "all_split": (0, N, N, 2 * N),
            "all_pruned": (0, 0, N, 0)}[case]
    assert (info["cloned"], info["split"], info["pruned"], info["n"]) == want


# ---------------------------------------------------------------------------------------------------------------------
# S5 image loss
# ---------------------------------------------------------------------------------------------------------------------
S5_CASES = [("random", 161, 161, 1.0), ("random", 161, 1000, 0.125), ("random", 163, 322, 1.0), ("random", 540, 960, 0.125),
            ("random", 1024, 1024, 1.0), ("random", 1080, 1920, 1.0), ("identical", 163, 322, 1.0), ("identical", 540, 960, 0.125),
            ("mask_zero", 163, 322, 1.0), ("mask_binary", 163, 322, 0.125), ("mask_soft", 540, 960, 1.0), ("clamp", 163, 322, 1.0),
            ("clamp", 1080, 1920, 0.125), ("anticorr", 163, 322, 1.0), ("anticorr", 540, 960, 0.125)]
S5_NO_SSIM = [(1, 1), (1, 37), (17, 3)]


def s5_inputs(content, H, W, seed=0):
    """img [5,H,W] (rgb | depth | alpha), ref [3,H,W], mask [1,H,W], fp32 on the CPU"""
    g = torch.Generator().manual_seed(seed + H * 7 + W + len(content))
    ref = torch.rand(3, H, W, generator=g)
    img = torch.cat([ref + 0.25 * torch.randn(3, H, W, generator=g), torch.rand(2, H, W, generator=g)])
    mask = torch.rand(1, H, W, generator=g)
    mask[:, :, : W // 3] = 1.0
    mask[:, H // 2:, W // 2:] = 0.0
    if content == "identical":
        img[:3] = ref; mask.fill_(1.0)
    elif content == "mask_zero":
        mask.zero_()
    elif content == "mask_binary":
        mask = (mask > 0.5).float()
    elif content == "clamp":
        mask.fill_(1.0)
        vals = torch.tensor([0.0, 1.0, f32_next(0.0, -1), f32_next(1.0, 1), f32_next(0.0, 1), f32_next(1.0, -1)])
        sel = torch.randint(0, vals.numel(), (3, H, W), generator=g)
        pick = torch.rand(3, H, W, generator=g) < 0.5
        img[:3] = torch.where(pick, vals[sel], img[:3])
    elif content == "anticorr":
        mask.fill_(1.0)
        img[0] = 1.0 - ref[0]
    return img.contiguous(), ref.contiguous(), mask.contiguous()


def loss_ref(img, ref, mask, ls, la, scale, dtype):
    """training_loss with the trainer's clamp, evaluated in `dtype` with autograd on the given (fp32) inputs"""
    from gs_b200 import losses
    x = img.to(dtype).clone().requires_grad_(True)
    loss = losses.training_loss(x[None, :3].clamp(0, 1), x[None, 4:5], ref.to(dtype)[None], mask.to(dtype)[None], ls, la) * scale
    loss.backward()
    return loss.detach(), x.grad


def check_loss(name, img, ref, mask, ls, la, scale):
    from gs_b200 import optim_step
    lk, dl = optim_step.image_loss(img, ref, mask, ls, la, scale)
    torch.cuda.synchronize()
    l64, g64 = loss_ref(img, ref, mask, ls, la, scale, torch.float64)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        l32, g32 = loss_ref(img, ref, mask, ls, la, scale, torch.float32)
    H, W = img.shape[1:]
    npix = H * W
    err_l = abs(float(lk) - float(l64))
    bar_l = K_LOSS * abs(float(l32) - float(l64)) + gam(10) * abs(float(l64))
    print(f"{name} loss: err {err_l:.3g}, err/bar {err_l / max(bar_l, 1e-300):.3g}, rel {err_l / max(abs(float(l64)), 1e-300):.3g}")
    assert err_l <= bar_l and err_l <= LOSS_VAL_REL * abs(float(l64)) + TINY, (name, err_l, bar_l)
    assert float(dl[3].abs().max()) == 0.0
    # L1 sign where |y - x| is a rounding decision
    x = (ref * mask).double(); y = (img[:3].clamp(0, 1) * mask).double()
    k1 = scale * (1 - ls) / (3.0 * npix)
    amb = ((y - x).abs() <= 4 * U * (x.abs() + y.abs())) & (img[:3] >= 0) & (img[:3] <= 1)
    unit = scale / (3.0 * npix)
    for c, pn in ((0, "r"), (1, "g"), (2, "b"), (4, "alpha")):
        err = (dl[c].double() - g64[c]).abs()
        if c < 3:
            err = (err - torch.where(amb[c], 2 * k1 * mask[0].double(), torch.zeros_like(err))).clamp_min(0)
        bar = K_LOSS * float((g32[c].double() - g64[c]).abs().max()) + TINY
        fixed = LOSS_GRAD_MAX * max(float(g64[c].abs().max()), unit)
        e = float(err.max())
        print(f"{name} plane {pn}: max err {e:.3g}, err/bar {e / bar:.3g}, err/fixed {e / fixed:.3g}")
        assert e <= bar and e <= fixed, (name, pn, e, bar, fixed)


@pytest.mark.gpu
@pytest.mark.parametrize("content,H,W,scale", S5_CASES)
def test_s5_image_loss(dev, content, H, W, scale):
    img, ref, mask = (t.to(dev) for t in s5_inputs(content, H, W))
    check_loss(f"S5 {content} {H}x{W} scale {scale}", img, ref, mask, 0.2, 3.0, scale)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", S5_NO_SSIM)
def test_s5_image_loss_without_ssim_at_tiny_shapes(dev, H, W):
    img, ref, mask = (t.to(dev) for t in s5_inputs("random", H, W))
    check_loss(f"S5 no-ssim {H}x{W}", img, ref, mask, 0.0, 3.0, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(160, 400), (400, 160), (160, 160)])
def test_s5_image_loss_refuses_sides_of_160(dev, H, W):
    from gs_b200 import optim_step
    img, ref, mask = (t.to(dev) for t in s5_inputs("random", H, W))
    with pytest.raises(RuntimeError, match="160"):
        optim_step.image_loss(img, ref, mask, 0.2, 3.0, 1.0)
    optim_step.image_loss(img, ref, mask, 0.0, 3.0, 1.0)           # without MS-SSIM any size is fine
