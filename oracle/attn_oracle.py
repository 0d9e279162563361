"""Float64 varlen multi-head attention, with the elementwise error bound of the fp16 / bf16 kernel (csrc/gs_attn.cu).

attention(q, k, v, cu_q, cu_k, scale) -> (out, bound), torch float64 on the inputs' device, so the GPU tests can run it
at caller sizes.  q [Tq, H, d], k / v [Tk, H, d] (any float dtype, taken as exact), cu_q / cu_k int [B + 1] or None
(one sequence).  out[i, h] = sum_j w_j v_j with w = softmax_j(scale * q_i . k_j) over the row's sequence; 0 without
keys.  Rows outside every sequence get out = 0 and bound = inf (the kernel does not write them).

The bound, with u the unit roundoff of the dtype (2^-11 fp16, 2^-8 bf16), e = 2^-24 that of fp32, n_k the sequence's
key count, sigma_i = scale * max_j sum_d |q_id| |k_jd| and A_i = sum_j w_j |v_j| (per output dim):

    |out_kernel - out| <= (2u + e (n_k + d sigma + c)) A + u |out| + tiny (sum_j |v_j| / l + 1),   c = 32

- P.  The kernel forms p_j = exp2(x_j - m) with x_j = fl(s_j * fl(scale log2 e)) in fp32.  The common shift m cancels
  in sum_j p_j v_j / sum_j p_j.  The fp32 error of s_j (four m16n8k16 accumulation steps over d = 64, each within a
  few units of 2^-24 sum |q||k|), the two roundings forming x_j and the one of x_j - m move p_j by a relative
  e (8 + 4) sigma_i at most; exp2f adds 2 ulp.  A relative error eta in every p_j moves out by at most 2 eta A (numerator
  and denominator): d sigma = 64 sigma covers 2 (8 + 4) sigma; c covers the exp2f, division and rescale terms.
- Rounding p to the dtype for P.V (the row sum l takes the unrounded p) moves out by u A; rounding out moves it by
  u |out|.  The bound charges 2u A for the first, which leaves room for the second-order terms.
- Sums.  P.V sums the exact dtype x dtype products in fp32 over n_k keys (n_k / 16 tensor-core steps plus one rescale
  per 64-key tile); l sums n_k / 4 values per lane, then rescales and a 4-lane reduction: e n_k covers both.
- Underflow.  p below the dtype's smallest normal is rounded with an absolute error of half its smallest subnormal
  (tiny = 2^-25 fp16, 2^-134 bf16; exp2f's flush of fp32 subnormals is below 2^-126 and is charged to tiny as well for
  bf16): in the final frame the error of out is at most tiny sum_j |v_j| / l, with l = sum_j exp(t_j - max t) >= 1.
  The same tiny bounds the rounding of a subnormal out.
"""
import math

import torch

C_BOUND = 32
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
TINY = {torch.float16: 2.0 ** -25, torch.bfloat16: 2.0 ** -125}


def _bounds(cu, total):
    if cu is None:
        return [(0, total)]
    c = [int(x) for x in cu.tolist()]
    out = []
    for b in range(len(c) - 1):
        s = min(max(c[b], 0), total)
        out.append((s, min(max(c[b + 1], s), total)))
    return out


def attention(q, k, v, cu_q=None, cu_k=None, scale=None, dtype=torch.float16):
    """(out, bound) in float64; `dtype` is the kernel's input dtype the bound is for."""
    d = q.shape[-1]
    scale = d ** -0.5 if scale is None else float(scale)
    q64, k64, v64 = q.double(), k.double(), v.double()
    Tq, H = q.shape[0], q.shape[1]
    out = torch.zeros(Tq, H, d, dtype=torch.float64, device=q.device)
    bound = torch.full((Tq, H, d), math.inf, dtype=torch.float64, device=q.device)
    u, tiny, e = U[dtype], TINY[dtype], 2.0 ** -24
    for (qs, qe), (ks, ke) in zip(_bounds(cu_q, Tq), _bounds(cu_k, k.shape[0])):
        if qe <= qs:
            continue
        nk = ke - ks
        if nk == 0:
            bound[qs:qe] = 0.0
            continue
        qb, kb, vb = q64[qs:qe].transpose(0, 1), k64[ks:ke].transpose(0, 1), v64[ks:ke].transpose(0, 1)  # [H, n, d]
        t = scale * qb @ kb.transpose(1, 2)                                     # [H, nq, nk]
        t = t - t.amax(-1, keepdim=True)
        p = torch.exp(t)
        lsum = p.sum(-1, keepdim=True)
        w = p / lsum
        o = w @ vb                                                              # [H, nq, d]
        a = w @ vb.abs()
        sigma = abs(scale) * (qb.abs() @ kb.abs().transpose(1, 2)).amax(-1, keepdim=True)
        under = tiny * (vb.abs().sum(1, keepdim=True) / lsum + 1.0)
        bnd = (2 * u + e * (nk + d * sigma + C_BOUND)) * a + u * o.abs() + under
        out[qs:qe] = o.transpose(0, 1)
        bound[qs:qe] = bnd.transpose(0, 1)
    return out, bound


def naive(q, k, v, cu_q=None, cu_k=None, scale=None):
    """The same attention as a per-row, per-head Python loop in float64 (to check attention() itself)."""
    d = q.shape[-1]
    scale = d ** -0.5 if scale is None else float(scale)
    out = torch.zeros(q.shape[0], q.shape[1], d, dtype=torch.float64)
    for (qs, qe), (ks, ke) in zip(_bounds(cu_q, q.shape[0]), _bounds(cu_k, k.shape[0])):
        for i in range(qs, qe):
            for h in range(q.shape[1]):
                if ke == ks:
                    continue
                logits = [scale * float(q[i, h].double() @ k[j, h].double()) for j in range(ks, ke)]
                mx = max(logits)
                ws = [math.exp(x - mx) for x in logits]
                tot = sum(ws)
                for j, wj in zip(range(ks, ke), ws):
                    out[i, h] += wj / tot * v[j, h].double()
    return out


def cu_from_lengths(lengths, device="cpu"):
    c = [0]
    for n in lengths:
        c.append(c[-1] + int(n))
    return torch.tensor(c, dtype=torch.int32, device=device)
