"""CPU tests of the flash_attn drop-in: the float64 oracle (oracle/attn_oracle.py) against torch's SDPA and a naive
loop; a numpy emulation of the kernel's fp32 / fp16 / bf16 rounding staying inside the oracle's bound on adversarial
logits (and coming close enough to it that the bound is not vacuous); the recorded fixture's self-consistency; the
shim's names and signatures; every argument error before any GPU work; the ABI through _lib."""
import inspect
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import attn_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_flash_attn.npz")
FUNCS = ["flash_attn_varlen_qkvpacked_func", "flash_attn_varlen_kvpacked_func", "flash_attn_varlen_func",
         "flash_attn_qkvpacked_func", "flash_attn_kvpacked_func", "flash_attn_func"]


def _fa():
    import flash_attn
    return flash_attn


# ---- oracle ---------------------------------------------------------------------------------------------------------
def test_oracle_matches_sdpa_per_sequence():
    g = torch.Generator().manual_seed(0)
    lq, lk = [5, 0, 33, 1], [7, 3, 0, 40]
    q = torch.randn(sum(lq), 3, 64, generator=g, dtype=torch.float64)
    k = torch.randn(sum(lk), 3, 64, generator=g, dtype=torch.float64)
    v = torch.randn(sum(lk), 3, 64, generator=g, dtype=torch.float64)
    cq, ck = O.cu_from_lengths(lq), O.cu_from_lengths(lk)
    out, bound = O.attention(q, k, v, cq, ck, scale=0.3)
    for b in range(len(lq)):
        qs, qe, ks, ke = int(cq[b]), int(cq[b + 1]), int(ck[b]), int(ck[b + 1])
        if qe == qs:
            continue
        if ke == ks:
            assert bool((out[qs:qe] == 0).all()) and bool((bound[qs:qe] == 0).all())
            continue
        ref = F.scaled_dot_product_attention(q[qs:qe].transpose(0, 1), k[ks:ke].transpose(0, 1),
                                             v[ks:ke].transpose(0, 1), scale=0.3).transpose(0, 1)
        assert torch.allclose(out[qs:qe], ref, rtol=1e-12, atol=1e-12)


def test_oracle_matches_naive_loop():
    g = torch.Generator().manual_seed(1)
    lq, lk = [3, 4, 0], [2, 0, 5]
    q = torch.randn(sum(lq), 2, 64, generator=g).half()
    k = torch.randn(sum(lk), 2, 64, generator=g).half()
    v = torch.randn(sum(lk), 2, 64, generator=g).half()
    cq, ck = O.cu_from_lengths(lq), O.cu_from_lengths(lk)
    out, _ = O.attention(q, k, v, cq, ck)
    assert torch.allclose(out, O.naive(q, k, v, cq, ck), rtol=1e-12, atol=1e-13)


def test_oracle_clamps_malformed_bounds():
    """cu_seqlens past the ends or decreasing are clamped as the kernel clamps them"""
    assert O._bounds(torch.tensor([-3, 4, 2, 99]), 10) == [(0, 4), (4, 4), (2, 10)]


# ---- emulation of the kernel's arithmetic ---------------------------------------------------------------------------
def _round(x, dtype):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dtype).float().numpy()


def emulate(q, k, v, dtype, scale=None):
    """one sequence, one head, as csrc/gs_attn.cu computes it: fp32 S, x = S * fl(scale log2 e), online softmax over
    64-key tiles on exp2, p rounded to the dtype for P.V, l over the unrounded p, out = O / l rounded once"""
    d = q.shape[-1]
    scale = d ** -0.5 if scale is None else scale
    sl2 = np.float32(scale * math.log2(math.e))
    f32 = np.float32
    m = np.full(q.shape[0], -np.inf, f32)
    lsum = np.zeros(q.shape[0], f32)
    o = np.zeros((q.shape[0], d), f32)
    q32, k32, v32 = q.astype(f32), k.astype(f32), v.astype(f32)
    for t0 in range(0, k.shape[0], 64):
        s = (q32 @ k32[t0:t0 + 64].T).astype(f32)
        x = (s * sl2).astype(f32)
        mx = np.maximum(m, x.max(1)).astype(f32)
        alpha = np.exp2((m - mx).astype(f32)).astype(f32)
        p = np.exp2((x - mx[:, None]).astype(f32)).astype(f32)
        lsum = (lsum * alpha + p.sum(1, dtype=f32)).astype(f32)
        o = (o * alpha[:, None] + _round(p, dtype) @ v32[t0:t0 + 64]).astype(f32)
        m = mx
    return _round(o / lsum[:, None], dtype)


def _adversarial(seed, dtype, nk, peak_scale):
    rng = np.random.default_rng(seed)
    q = _round(rng.standard_normal((48, 64)) * peak_scale, dtype)
    k = _round(rng.standard_normal((nk, 64)) * peak_scale, dtype)
    v = _round(rng.standard_normal((nk, 64)), dtype)
    k[-3:] = _round(q[:3] * 1.25, dtype)             # rows 0..2 peak in the last tile
    k[nk // 2] = _round(q[3] * 1.25, dtype)          # row 3 peaks in a middle tile
    k[-10:-3] = _round(q[4:5] * 1.2 + rng.standard_normal((7, 64)) * 0.01, dtype)  # near-ties for row 4
    v[-1] *= 1e-3                                    # a small value under the largest weight
    return q, k, v


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nk,peak", [(300, 1.0), (1000, 6.0), (700, 0.05), (4100, 2.5)])
def test_emulation_inside_bound(dtype, nk, peak):
    q, k, v = _adversarial(nk, dtype, nk, peak)
    got = emulate(q, k, v, dtype)
    ref, bound = O.attention(torch.from_numpy(q)[:, None], torch.from_numpy(k)[:, None], torch.from_numpy(v)[:, None],
                             dtype=dtype)
    err = np.abs(got.astype(np.float64) - ref[:, 0].numpy())
    ratio = err / bound[:, 0].numpy()
    assert ratio.max() <= 1.0, f"emulated error exceeds the bound: ratio {ratio.max():.3f}"
    # not vacuous: the rounding that the bound charges with u is reached to within a small factor
    assert ratio.max() >= 0.02, f"bound is loose by {1 / ratio.max():.0f}x"


# ---- fixture --------------------------------------------------------------------------------------------------------
def test_fixture_self_consistent():
    z = np.load(GOLDEN)
    cases = sorted({k.split("/")[0] for k in z.files})
    fns = [FUNCS[int(z[f"{c}/fn"])] for c in cases]
    assert {"flash_attn_varlen_qkvpacked_func", "flash_attn_varlen_kvpacked_func", "flash_attn_kvpacked_func",
            "flash_attn_func"} <= set(fns)
    assert fns.count("flash_attn_varlen_qkvpacked_func") == 3    # full, windowed shift 0, windowed shift 4
    for c, fn in zip(cases, fns):
        dtype = torch.bfloat16 if int(z[f"{c}/bf16"]) else torch.float16
        assert dtype == (torch.bfloat16 if fn == "flash_attn_func" and int(z[f"{c}/bf16"]) else torch.float16)
        tensors = [torch.from_numpy(z[f"{c}/arg{i}"]).view(dtype) for i in range(int(z[f"{c}/n_args"]))]
        cus = [torch.from_numpy(z[f"{c}/cu{i}"]) for i in range(int(z[f"{c}/n_cu"]))]
        ints = [int(x) for x in z[f"{c}/ints"]]
        for cu in cus:
            assert cu.dtype == torch.int32 and int(cu[0]) == 0 and bool((cu[1:] >= cu[:-1]).all())
        assert ints == [int((cu[1:] - cu[:-1]).max()) for cu in (cus * 2 if len(cus) == 1 and ints else cus)][:len(ints)]
        out = torch.from_numpy(z[f"{c}/out"])
        if fn == "flash_attn_varlen_qkvpacked_func":
            q, k, v = tensors[0].unbind(1)
            ref = O.attention(q, k, v, cus[0], cus[0])[0]
        elif fn == "flash_attn_varlen_kvpacked_func":
            q, (k, v) = tensors[0], tensors[1].unbind(1)
            ref = O.attention(q, k, v, cus[0], cus[1])[0]
        else:
            if fn == "flash_attn_kvpacked_func":
                q, (k, v) = tensors[0], tensors[1].unbind(2)
            else:
                q, k, v = tensors
            ref = torch.stack([O.attention(q[b], k[b], v[b])[0] for b in range(q.shape[0])])
        assert torch.equal(out, ref)
        assert out.shape[-2:] == (q.shape[-2], 64)


# ---- shim -----------------------------------------------------------------------------------------------------------
SIGS = {
    "flash_attn_varlen_qkvpacked_func": ["qkv", "cu_seqlens", "max_seqlen"],
    "flash_attn_varlen_kvpacked_func": ["q", "kv", "cu_seqlens_q", "cu_seqlens_k", "max_seqlen_q", "max_seqlen_k"],
    "flash_attn_varlen_func": ["q", "k", "v", "cu_seqlens_q", "cu_seqlens_k", "max_seqlen_q", "max_seqlen_k"],
    "flash_attn_qkvpacked_func": ["qkv"],
    "flash_attn_kvpacked_func": ["q", "kv"],
    "flash_attn_func": ["q", "k", "v"],
}
COMMON = ["dropout_p", "softmax_scale", "causal", "window_size", "softcap", "alibi_slopes", "deterministic",
          "return_attn_probs"]


def test_shim_names_and_signatures():
    fa = _fa()
    assert fa.__version__.startswith("2.")
    assert sorted(fa.__all__) == sorted(SIGS)
    for name, pos in SIGS.items():
        params = list(inspect.signature(getattr(fa, name)).parameters.values())
        names = [p.name for p in params]
        extra = ["block_table"] if name == "flash_attn_varlen_func" else []
        assert names == pos + COMMON + extra, name
        defaults = {p.name: p.default for p in params}
        assert defaults["dropout_p"] == 0.0 and defaults["softmax_scale"] is None and defaults["causal"] is False
        assert defaults["window_size"] == (-1, -1) and defaults["return_attn_probs"] is False


def test_shim_is_this_projects_and_ships_no_metadata():
    """`import flash_attn` resolves to the shim, which carries no dist-info / egg-info of its own"""
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    shim_dir = os.path.join(here, "comfyui-3d-pack_b200", "flash_attn")
    assert os.path.dirname(os.path.abspath(_fa().__file__)) == shim_dir
    pkg = os.path.dirname(shim_dir)
    assert not [f for f in os.listdir(pkg) if f.startswith("flash_attn") and f.endswith(("-info", ".pth"))]


def _t(*shape, dtype=torch.float16):
    return torch.zeros(*shape, dtype=dtype)


def _cu(*vals, dtype=torch.int32):
    return torch.tensor(vals, dtype=dtype)


@pytest.mark.parametrize("kw,word", [({"dropout_p": 0.1}, "dropout_p"), ({"causal": True}, "causal"),
                                     ({"window_size": (8, 8)}, "window_size"), ({"softcap": 30.0}, "softcap"),
                                     ({"alibi_slopes": _t(2)}, "alibi_slopes"),
                                     ({"return_attn_probs": True}, "return_attn_probs")])
def test_unsupported_arguments(kw, word):
    fa = _fa()
    calls = [lambda: fa.flash_attn_varlen_qkvpacked_func(_t(4, 3, 2, 64), _cu(0, 4), 4, **kw),
             lambda: fa.flash_attn_varlen_kvpacked_func(_t(4, 2, 64), _t(4, 2, 2, 64), _cu(0, 4), _cu(0, 4), 4, 4, **kw),
             lambda: fa.flash_attn_varlen_func(_t(4, 2, 64), _t(4, 2, 64), _t(4, 2, 64), _cu(0, 4), _cu(0, 4), 4, 4,
                                               **kw),
             lambda: fa.flash_attn_qkvpacked_func(_t(1, 4, 3, 2, 64), **kw),
             lambda: fa.flash_attn_kvpacked_func(_t(1, 4, 2, 64), _t(1, 4, 2, 2, 64), **kw),
             lambda: fa.flash_attn_func(_t(1, 4, 2, 64), _t(1, 4, 2, 64), _t(1, 4, 2, 64), **kw)]
    for call in calls:
        with pytest.raises(NotImplementedError, match=word):
            call()
    with pytest.raises(NotImplementedError, match="block_table"):
        fa.flash_attn_varlen_func(_t(4, 2, 64), _t(4, 2, 64), _t(4, 2, 64), _cu(0, 4), _cu(0, 4), 4, 4,
                                  block_table=_cu(0))


def test_argument_errors_before_gpu_work():
    fa = _fa()
    q, kv = _t(4, 2, 64), _t(4, 2, 2, 64)
    # dtype
    with pytest.raises(TypeError):
        fa.flash_attn_func(_t(1, 4, 2, 64, dtype=torch.float32), _t(1, 4, 2, 64), _t(1, 4, 2, 64))
    with pytest.raises(TypeError, match="mixed"):
        fa.flash_attn_func(_t(1, 4, 2, 64, dtype=torch.bfloat16), _t(1, 4, 2, 64), _t(1, 4, 2, 64))
    with pytest.raises(TypeError):
        fa.flash_attn_varlen_qkvpacked_func(_t(4, 3, 2, 64, dtype=torch.float64), _cu(0, 4), 4)
    # shapes
    with pytest.raises(NotImplementedError, match="head dim"):
        fa.flash_attn_func(_t(1, 4, 2, 128), _t(1, 4, 2, 128), _t(1, 4, 2, 128))
    with pytest.raises(NotImplementedError, match="kv heads"):
        fa.flash_attn_kvpacked_func(_t(1, 4, 4, 64), _t(1, 4, 2, 2, 64))
    with pytest.raises(ValueError):
        fa.flash_attn_varlen_qkvpacked_func(_t(4, 2, 2, 64), _cu(0, 4), 4)
    with pytest.raises(ValueError):
        fa.flash_attn_func(_t(4, 2, 64), _t(4, 2, 64), _t(4, 2, 64))
    with pytest.raises(ValueError):
        fa.flash_attn_func(_t(2, 4, 2, 64), _t(1, 4, 2, 64), _t(1, 4, 2, 64))
    with pytest.raises(ValueError, match="int32"):
        fa.flash_attn_varlen_kvpacked_func(q, kv, _cu(0, 4, dtype=torch.int64), _cu(0, 4), 4, 4)
    with pytest.raises(ValueError):
        fa.flash_attn_varlen_kvpacked_func(q, kv, _cu(0, 2, 4), _cu(0, 4), 4, 4)
    with pytest.raises(ValueError):
        fa.flash_attn_varlen_kvpacked_func(q, kv, _cu(0, 4), _cu(0, 4), -1, 4)
    # device: valid arguments on the CPU
    with pytest.raises(RuntimeError, match="CPU"):
        fa.flash_attn_varlen_kvpacked_func(q, kv, _cu(0, 4), _cu(0, 4), 4, 4)
    with pytest.raises(RuntimeError, match="CPU"):
        fa.flash_attn_func(_t(1, 4, 2, 64, dtype=torch.bfloat16), _t(1, 4, 2, 64, dtype=torch.bfloat16),
                           _t(1, 4, 2, 64, dtype=torch.bfloat16))


# ---- ABI ------------------------------------------------------------------------------------------------------------
def test_abi_is_bound_from_include_with_its_constants():
    """gs_b200_attn_forward is bound from include/gs_b200_attn.h, with its constants; its argument errors are reported
    through gs_b200_last_error"""
    import ctypes as C
    from gs_b200 import _lib
    assert (_lib.ATTN_F16, _lib.ATTN_BF16, _lib.ATTN_HEAD_DIM) == (0, 1, 64)
    header = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gs_b200_attn.h")
    protos = _lib.prototypes(open(header).read())
    assert list(protos) == ["gs_b200_attn_forward"]
    import subprocess
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-x", "c", header], check=True)
    fn = _lib.lib.gs_b200_attn_forward
    assert fn.restype is C.c_int32 and len(fn.argtypes) == 22
    assert fn.argtypes[19] is C.c_float
    # invalid arguments are refused before any launch, with a message
    assert fn(7, 1, 1, 64, None, 0, 0, None, 0, 0, None, 0, 0, None, None, 1, 1, 1, 1, C.c_float(1.0), None, None) == 1
    assert "dtype" in _lib.last_error()
    assert fn(0, 1, 1, 32, None, 0, 0, None, 0, 0, None, 0, 0, None, None, 1, 1, 1, 1, C.c_float(1.0), None, None) == 1
    assert "head dim" in _lib.last_error()
    assert fn(0, 2, 1, 64, None, 0, 0, None, 0, 0, None, 0, 0, None, None, 3, 3, 5, 6, C.c_float(1.0), None, None) == 1
    assert "B * max_seqlen" in _lib.last_error()
