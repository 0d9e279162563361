"""Generates tests/golden/ref_flash_attn.npz by running the REFERENCE's own flash_attn callers on the CPU, with this
project's `flash_attn` shim imported and its six functions wrapped by recorders that compute with
oracle/attn_oracle.py (float64) and check every call against the shim's signatures.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python tests/golden/make_golden_flash_attn.py

TRELLIS's trellis/__init__.py pulls in ComfyUI, so a bare `trellis` package is registered whose __path__ is the
reference's trellis/ directory, with ATTN_BACKEND=flash_attn set before the import, as a TRELLIS user sets it.
Callers run in fp16 (TRELLIS) with seeded weights, channels 128 = 2 heads of 64:
  1. SparseMultiHeadAttention, full self-attention with qk_rms_norm (the SLat flow), two batch items of 20 and 50 voxels.
  2. The same module in windowed mode (the SLat decoders' swin blocks): window 8, shift (0,0,0) and (4,4,4).
  3. SparseMultiHeadAttention cross-attention from those voxels to a dense [2, 13, 96] context.
  4. MultiHeadAttention (dense) self-attention on [2, 24, 128] and cross-attention to [2, 13, 96].
  5. Hunyuan3D 1.0's FlashAttention (its own bf16 cast), query [1, 24, 128], 2 heads.
For each call the file holds, under call<NNN>/: the function (index into FUNCS), the dtype (bf16 flag), the tensor
arguments as int16 bits, the int32 cu_seqlens, the max_seqlen ints, the keyword arguments as numbers (dropout_p,
softmax_scale or NaN for None, causal) and the float64 result.  Nothing from the reference is stored: only numbers.
"""
import inspect
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.join(ROOT, "comfyui-3d-pack_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)
from oracle import attn_oracle as O  # noqa: E402

REF = os.environ["COMFYUI_3D_PACK"]
MODS = os.path.join(REF, "Gen_3D_Modules")
FUNCS = ["flash_attn_varlen_qkvpacked_func", "flash_attn_varlen_kvpacked_func", "flash_attn_varlen_func",
         "flash_attn_qkvpacked_func", "flash_attn_kvpacked_func", "flash_attn_func"]
CALLS = []


def _compute(fn, tensors, cus):
    if fn.startswith("flash_attn_varlen"):
        if fn == "flash_attn_varlen_qkvpacked_func":
            (q, k, v), cq, ck = tensors[0].unbind(1), cus[0], cus[0]
        elif fn == "flash_attn_varlen_kvpacked_func":
            (q, (k, v)), (cq, ck) = (tensors[0], tensors[1].unbind(1)), cus
        else:
            (q, k, v), (cq, ck) = tensors, cus
        return O.attention(q, k, v, cq, ck)[0]
    if fn == "flash_attn_qkvpacked_func":
        q, k, v = tensors[0].unbind(2)
    elif fn == "flash_attn_kvpacked_func":
        q, (k, v) = tensors[0], tensors[1].unbind(2)
    else:
        q, k, v = tensors
    return torch.stack([O.attention(q[b], k[b], v[b])[0] for b in range(q.shape[0])])


def _recorder(shim, fn):
    sig = inspect.signature(getattr(shim, fn))

    def rec(*args, **kwargs):
        bound = sig.bind(*args, **kwargs)            # the caller's arguments fit the shim's signature
        bound.apply_defaults()
        a = bound.arguments
        assert a["dropout_p"] == 0.0 and not a["causal"] and tuple(a["window_size"]) == (-1, -1)
        tensors = [x for x in args if isinstance(x, torch.Tensor) and x.dtype != torch.int32]
        cus = [x for x in args if isinstance(x, torch.Tensor) and x.dtype == torch.int32]
        ints = [int(x) for x in args if not isinstance(x, torch.Tensor)]
        assert all(isinstance(x, int) for x in args if not isinstance(x, torch.Tensor)), "max_seqlen must be an int"
        dtype = tensors[0].dtype
        out = _compute(fn, tensors, cus)
        scale = a["softmax_scale"]
        CALLS.append({"fn": np.int32(FUNCS.index(fn)), "bf16": np.int32(dtype == torch.bfloat16),
                      "n_args": np.int32(len(tensors)), "n_cu": np.int32(len(cus)),
                      "ints": np.array(ints, dtype=np.int64),
                      "kw": np.array([a["dropout_p"], np.nan if scale is None else scale, float(a["causal"])]),
                      "out": out.numpy(),
                      **{f"arg{i}": t.contiguous().view(torch.int16).numpy() for i, t in enumerate(tensors)},
                      **{f"cu{i}": c.numpy() for i, c in enumerate(cus)}})
        return out.to(dtype)
    return rec


def main():
    os.environ["ATTN_BACKEND"] = "flash_attn"
    os.environ["SPARSE_BACKEND"] = "spconv"
    import flash_attn as shim
    assert os.path.dirname(shim.__file__) == os.path.join(ROOT, "comfyui-3d-pack_b200", "flash_attn"), shim.__file__
    for fn in FUNCS:
        setattr(shim, fn, _recorder(shim, fn))

    pkg = types.ModuleType("trellis")
    pkg.__path__ = [os.path.join(MODS, "TRELLIS", "trellis")]
    sys.modules["trellis"] = pkg
    from trellis.modules import sparse as sp
    from trellis.modules.sparse.attention import SparseMultiHeadAttention
    from trellis.modules.attention import MultiHeadAttention
    assert sp.ATTN == "flash_attn"

    torch.manual_seed(0)
    g = torch.Generator().manual_seed(1)
    C, H = 128, 2
    coords = [torch.randint(0, 16, (n, 3), generator=g) for n in (20, 50)]
    coords = [torch.unique(c, dim=0) for c in coords]
    coords = torch.cat([torch.cat([torch.full((c.shape[0], 1), b), c], 1) for b, c in enumerate(coords)]).int()
    feats = torch.randn(coords.shape[0], C, generator=g).half()
    x = sp.SparseTensor(feats, coords)
    ctx = torch.randn(2, 13, 96, generator=g).half()
    with torch.no_grad():
        SparseMultiHeadAttention(C, H, type="self", attn_mode="full", qk_rms_norm=True).half()(x)
        for shift in ((0, 0, 0), (4, 4, 4)):
            SparseMultiHeadAttention(C, H, type="self", attn_mode="windowed", window_size=8,
                                     shift_window=shift).half()(x)
        SparseMultiHeadAttention(C, H, ctx_channels=96, type="cross", attn_mode="full").half()(x, ctx)
        xd = torch.randn(2, 24, C, generator=g).half()
        MultiHeadAttention(C, H, type="self", qk_rms_norm=True).half()(xd)
        MultiHeadAttention(C, H, ctx_channels=96, type="cross").half()(xd, ctx)

        import importlib.util
        spec = importlib.util.spec_from_file_location(
            "hy_attention", os.path.join(MODS, "Hunyuan3D_V1", "svrm", "ldm", "modules", "attention.py"))
        hy = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(hy)
        assert hy.FLASH_IS_AVAILABLE
        hy.FlashAttention(C, heads=H, dim_head=64)(torch.randn(1, 24, C, generator=g))

    fns = [FUNCS[int(c["fn"])] for c in CALLS]
    print(len(CALLS), "calls:", {f: fns.count(f) for f in FUNCS})
    arrays = {f"call{i:03d}/{k}": v for i, c in enumerate(CALLS) for k, v in c.items()}
    np.savez_compressed(os.path.join(HERE, "ref_flash_attn.npz"), **arrays)


if __name__ == "__main__":
    main()
