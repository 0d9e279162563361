"""GPU tests of the flash_attn drop-in (gs_b200.attention, csrc/gs_attn.cu) against the float64 oracle
(oracle/attn_oracle.py): every output must lie within the oracle's elementwise bound for the kernel's arithmetic, and
the outputs that the kernel's rules say are equal must have the same bits."""
import os

import numpy as np
import pytest
import torch

from oracle import attn_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_flash_attn.npz")
DTYPES = [torch.float16, torch.bfloat16]


def _fa():
    import flash_attn
    return flash_attn


def _rand(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(dtype)


def _within(got, q, k, v, cu_q=None, cu_k=None, scale=None, dtype=torch.float16):
    ref, bound = O.attention(q, k, v, cu_q, cu_k, scale, dtype)
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), (f"{int(bad.sum())} outputs outside the bound; worst err {float(err.max()):.3e}, "
                                 f"err / bound {float((err / bound).max()):.3f}")
    return float((err / bound.clamp_min(1e-300)).max())


def _same(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "bits differ"


# ---- lengths --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("L", [1, 63, 64, 65, 127, 129, 4096])
def test_lengths_varlen(dtype, L):
    lq, lk = [L, 7, 130], [L, 130, 7]
    H = 3
    q = _rand((sum(lq), H, 64), dtype, 1)
    k = _rand((sum(lk), H, 64), dtype, 2)
    v = _rand((sum(lk), H, 64), dtype, 3)
    cq, ck = O.cu_from_lengths(lq, DEV), O.cu_from_lengths(lk, DEV)
    out = _fa().flash_attn_varlen_func(q, k, v, cq, ck, max(lq), max(lk))
    _within(out, q, k, v, cq, ck, dtype=dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_empty_sequences(dtype):
    lq, lk = [5, 0, 70, 3], [9, 4, 0, 66]
    q = _rand((sum(lq), 2, 64), dtype, 4)
    k = _rand((sum(lk), 2, 64), dtype, 5)
    v = _rand((sum(lk), 2, 64), dtype, 6)
    cq, ck = O.cu_from_lengths(lq, DEV), O.cu_from_lengths(lk, DEV)
    out = _fa().flash_attn_varlen_func(q, k, v, cq, ck, max(lq), max(lk))
    assert bool((out[5:75] == 0).all()), "a sequence without keys must give 0"
    _within(out, q, k, v, cq, ck, dtype=dtype)
    # no query rows at all, and no key rows at all
    e = _fa().flash_attn_varlen_func(q[:0], k, v, torch.zeros(2, dtype=torch.int32, device=DEV),
                                     torch.tensor([0, 9], dtype=torch.int32, device=DEV), 0, 9)
    assert e.shape == (0, 2, 64)
    z = _fa().flash_attn_varlen_func(q[:5], k[:0], v[:0], torch.tensor([0, 5], dtype=torch.int32, device=DEV),
                                     torch.zeros(2, dtype=torch.int32, device=DEV), 5, 0)
    assert bool((z == 0).all())


@pytest.mark.parametrize("dtype", DTYPES)
def test_windows(dtype):
    """thousands of 1..512-row windows, as TRELLIS's windowed self-attention packs them (qkv packed, H 12)"""
    rng = np.random.default_rng(7)
    lens = rng.integers(1, 513, size=2000)
    lens[:8] = [1, 512, 64, 65, 1, 2, 511, 63]
    qkv = _rand((int(lens.sum()), 3, 12, 64), dtype, 8)
    cu = O.cu_from_lengths(lens, DEV)
    out = _fa().flash_attn_varlen_qkvpacked_func(qkv, cu, int(lens.max()))
    q, k, v = qkv.unbind(1)
    _within(out, q, k, v, cu, cu, dtype=dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_long_sequence_sampled(dtype):
    """one 12 536-row sequence (the SLat flow's self-attention at 64^3), H 16; heads and rows sampled"""
    T, H = 12536, 16
    qkv = _rand((T, 3, H, 64), dtype, 9)
    cu = torch.tensor([0, T], dtype=torch.int32, device=DEV)
    out = _fa().flash_attn_varlen_qkvpacked_func(qkv, cu, T)
    rows = torch.cat([torch.arange(0, 70, device=DEV), torch.randperm(T, device=DEV)[:400],
                      torch.arange(T - 70, T, device=DEV)])
    heads = torch.tensor([0, 5, 15], device=DEV)
    q, k, v = qkv.unbind(1)
    _within(out[rows][:, heads], q[rows][:, heads], k[:, heads], v[:, heads], dtype=dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_many_one_row_sequences(dtype):
    """70 000 one-row sequences: more than 65 535 grid rows; each output is its own value row, exactly"""
    n = 70000
    qkv = _rand((n, 3, 2, 64), dtype, 10)
    cu = torch.arange(n + 1, dtype=torch.int32, device=DEV)
    out = _fa().flash_attn_varlen_qkvpacked_func(qkv, cu, 1)
    _same(out, qkv[:, 2].contiguous())


# ---- numerics -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_large_logits_late_max(dtype):
    """|s| ~ 10^3 with each row's maximum in the last key tile: the running max is replaced after many tiles"""
    lk, H = 1000, 4
    q = _rand((64, H, 64), dtype, 11, 8.0)
    k = _rand((lk, H, 64), dtype, 12, 8.0)
    v = _rand((lk, H, 64), dtype, 13)
    k[-5:] = (q[:5] * 1.5).to(dtype)            # rows 0..4 peak at keys lk-5..lk-1 (tile 15 of 16)
    k[-40] = -k[-40]
    cq = torch.tensor([0, 64], dtype=torch.int32, device=DEV)
    ck = torch.tensor([0, lk], dtype=torch.int32, device=DEV)
    out = _fa().flash_attn_varlen_func(q, k, v, cq, ck, 64, lk)
    s = (q.double()[:5] * k.double()[-5:]).sum(-1) / 8
    assert float(s.abs().min()) > 100
    _within(out, q, k, v, cq, ck, dtype=dtype)


# ---- bits -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_bits(dtype):
    fa = _fa()
    lens = [300, 1, 64, 129, 77]
    qkv = _rand((sum(lens), 3, 4, 64), dtype, 14)
    cu = O.cu_from_lengths(lens, DEV)
    ref = fa.flash_attn_varlen_qkvpacked_func(qkv, cu, max(lens))
    # every run
    for _ in range(3):
        _same(fa.flash_attn_varlen_qkvpacked_func(qkv, cu, max(lens)), ref)
    # a hint of 1 for max_seqlen
    _same(fa.flash_attn_varlen_qkvpacked_func(qkv, cu, 1), ref)
    # explicit and default softmax_scale
    _same(fa.flash_attn_varlen_qkvpacked_func(qkv, cu, max(lens), softmax_scale=64 ** -0.5), ref)
    # packed and unpacked, in-place strided and contiguous copies
    q, k, v = qkv.unbind(1)
    _same(fa.flash_attn_varlen_func(q, k, v, cu, cu, max(lens), max(lens)), ref)
    _same(fa.flash_attn_varlen_func(q.contiguous(), k.contiguous(), v.contiguous(), cu, cu, max(lens), max(lens)), ref)
    _same(fa.flash_attn_varlen_kvpacked_func(q, qkv[:, 1:], cu, cu, max(lens), max(lens)), ref)
    # a sequence alone and inside the batch
    s0, s1 = 365, 365 + 129
    alone = fa.flash_attn_varlen_qkvpacked_func(qkv[s0:s1].clone(), torch.tensor([0, 129], dtype=torch.int32,
                                                                                 device=DEV), 129)
    _same(alone, ref[s0:s1])


@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_equals_uniform_varlen(dtype):
    fa = _fa()
    N, L, H = 3, 200, 4
    qkv = _rand((N, L, 3, H, 64), dtype, 15)
    dense = fa.flash_attn_qkvpacked_func(qkv)
    cu = torch.arange(0, N * L + 1, L, dtype=torch.int32, device=DEV)
    var = fa.flash_attn_varlen_qkvpacked_func(qkv.reshape(N * L, 3, H, 64), cu, L)
    _same(dense.reshape(N * L, H, 64), var)
    q, k, v = qkv.unbind(2)
    _same(fa.flash_attn_func(q, k, v), dense)
    _same(fa.flash_attn_kvpacked_func(q, qkv[:, :, 1:]), dense)
    _same(fa.flash_attn_func(q.contiguous(), k.contiguous(), v.contiguous()), dense)
    _within(var, *qkv.reshape(N * L, 3, H, 64).unbind(1), cu, cu, dtype=dtype)


def test_dense_cross_and_hunyuan_shape():
    fa = _fa()
    q = _rand((2, 4096, 16, 64), torch.float16, 16)
    kv = _rand((2, 1374, 2, 16, 64), torch.float16, 17)
    out = fa.flash_attn_kvpacked_func(q, kv)
    assert out.shape == q.shape
    k, v = kv.unbind(2)
    sl = slice(0, 256)
    _within(out[1, sl], q[1, sl], k[1], v[1])
    qb, kb, vb = (_rand((1, 3079, 16, 64), torch.bfloat16, s) for s in (18, 19, 20))
    ob = fa.flash_attn_func(qb, kb, vb, dropout_p=0.0, softmax_scale=None, causal=False)
    _within(ob[0, ::7], qb[0, ::7], kb[0], vb[0], dtype=torch.bfloat16)


# ---- environment ----------------------------------------------------------------------------------------------------
def test_inference_grad_mode_and_side_stream():
    fa = _fa()
    qkv = _rand((150, 3, 2, 64), torch.float16, 21)
    cu = torch.tensor([0, 50, 150], dtype=torch.int32, device=DEV)
    ref = fa.flash_attn_varlen_qkvpacked_func(qkv, cu, 100)
    with torch.inference_mode():
        _same(fa.flash_attn_varlen_qkvpacked_func(qkv, cu, 100), ref)
    x = qkv.clone().requires_grad_(True)
    out = fa.flash_attn_varlen_qkvpacked_func(x, cu, 100)
    _same(out.detach(), ref)
    assert out.requires_grad
    with pytest.raises(NotImplementedError):
        out.float().sum().backward()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        o2 = fa.flash_attn_varlen_qkvpacked_func(qkv, cu, 100)
    torch.cuda.current_stream().wait_stream(s)
    _same(o2, ref)


# ---- the recorded reference calls ------------------------------------------------------------------------------------
FUNCS = ["flash_attn_varlen_qkvpacked_func", "flash_attn_varlen_kvpacked_func", "flash_attn_varlen_func",
         "flash_attn_qkvpacked_func", "flash_attn_kvpacked_func", "flash_attn_func"]


def _replay_cases():
    with np.load(GOLDEN) as z:
        return sorted({k.split("/")[0] for k in z.files if k.startswith("call")})


@pytest.mark.parametrize("case", _replay_cases() if os.path.exists(GOLDEN) else ["missing"])
def test_replay_recorded_calls(case):
    """every flash_attn call that TRELLIS's attention modules and Hunyuan3D 1.0's FlashAttention made while the
    fixture was recorded, replayed with the same argument bits, within the oracle's bound of the recorded result"""
    fa = _fa()
    z = np.load(GOLDEN)
    fn = FUNCS[int(z[f"{case}/fn"])]
    dtype = torch.bfloat16 if int(z[f"{case}/bf16"]) else torch.float16

    def arg(i):
        return torch.from_numpy(z[f"{case}/arg{i}"]).to(DEV).view(dtype)

    tensors = [arg(i) for i in range(int(z[f"{case}/n_args"]))]
    ints = [int(x) for x in z[f"{case}/ints"]]
    cus = [torch.from_numpy(z[f"{case}/cu{i}"]).to(DEV) for i in range(int(z[f"{case}/n_cu"]))]
    dropout_p, scale, causal = (float(x) for x in z[f"{case}/kw"])
    kw = {"dropout_p": dropout_p, "softmax_scale": None if np.isnan(scale) else scale, "causal": bool(causal)}
    expect = torch.from_numpy(z[f"{case}/out"]).to(DEV)
    out = getattr(fa, fn)(*tensors, *cus, *ints, **kw)
    assert out.shape == expect.shape
    if fn.startswith("flash_attn_varlen"):
        if fn == "flash_attn_varlen_qkvpacked_func":
            q, k, v = tensors[0].unbind(1)
            cq = ck = cus[0]
        elif fn == "flash_attn_varlen_kvpacked_func":
            q, (k, v) = tensors[0], tensors[1].unbind(1)
            cq, ck = cus
        else:
            q, k, v = tensors
            cq, ck = cus
        ref, bound = O.attention(q, k, v, cq, ck, kw["softmax_scale"], dtype)
    else:
        if fn == "flash_attn_qkvpacked_func":
            q, k, v = tensors[0].unbind(2)
        elif fn == "flash_attn_kvpacked_func":
            q, (k, v) = tensors[0], tensors[1].unbind(2)
        else:
            q, k, v = tensors
        refs = [O.attention(q[b], k[b], v[b], None, None, kw["softmax_scale"], dtype) for b in range(q.shape[0])]
        ref, bound = torch.stack([r[0] for r in refs]), torch.stack([r[1] for r in refs])
    assert torch.allclose(ref, expect.double(), rtol=1e-9, atol=1e-12), "the fixture's result is not the oracle's"
    err = (out.double() - ref).abs()
    assert bool((err <= bound).all()), f"worst err {float(err.max()):.3e}"
