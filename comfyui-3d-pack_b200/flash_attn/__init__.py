"""Import-name shim for the part of flash-attn 2.x that TRELLIS, Stable3DGen and Hunyuan3D 1.0 call: the six forward
functions below, under flash-attn 2.x's signatures, for head dim 64 in fp16 and bf16.  Attention runs on the GPU
through gs_b200.attention, which states the rules.  Differences from the package: forward only (a .backward() through
the output raises NotImplementedError); no CPU path; every output has the same bits on every run, so `deterministic`
is accepted and changes nothing.  dropout_p > 0, causal=True, a window_size other than (-1, -1), softcap != 0,
alibi_slopes, return_attn_probs=True and block_table raise NotImplementedError naming the argument; head dims other
than 64 and fewer kv heads than query heads raise NotImplementedError too.  With this directory on sys.path,
`import flash_attn` resolves here for the whole process, shadowing an installed flash-attn.  No distribution metadata
ships with it, so importlib.metadata lookups (transformers' and diffusers' availability probes) do not find it.
"""
from gs_b200 import attention as _A

__version__ = "2.7.3"

__all__ = ["flash_attn_func", "flash_attn_kvpacked_func", "flash_attn_qkvpacked_func", "flash_attn_varlen_func",
           "flash_attn_varlen_kvpacked_func", "flash_attn_varlen_qkvpacked_func"]


def _unsupported(name, dropout_p, causal, window_size, softcap, alibi_slopes, return_attn_probs, block_table=None):
    if dropout_p:
        raise NotImplementedError(f"{name}: dropout_p={dropout_p} (only 0.0 is implemented)")
    if causal:
        raise NotImplementedError(f"{name}: causal=True (only causal=False is implemented)")
    if window_size is not None and tuple(window_size) != (-1, -1):
        raise NotImplementedError(f"{name}: window_size={tuple(window_size)} (only (-1, -1) is implemented)")
    if softcap:
        raise NotImplementedError(f"{name}: softcap={softcap} (only 0.0 is implemented)")
    if alibi_slopes is not None:
        raise NotImplementedError(f"{name}: alibi_slopes is not implemented")
    if return_attn_probs:
        raise NotImplementedError(f"{name}: return_attn_probs=True is not implemented")
    if block_table is not None:
        raise NotImplementedError(f"{name}: block_table (paged KV cache) is not implemented")


def _split(name, packed, n, arg):
    if not hasattr(packed, "dim") or packed.dim() < 3 or packed.size(-3) != n:
        raise ValueError(f"{name}: {arg} must have {n} at dim -3, got shape {tuple(getattr(packed, 'shape', ()))}")
    return packed.unbind(-3)


def flash_attn_varlen_qkvpacked_func(qkv, cu_seqlens, max_seqlen, dropout_p=0.0, softmax_scale=None, causal=False,
                                     window_size=(-1, -1), softcap=0.0, alibi_slopes=None, deterministic=False,
                                     return_attn_probs=False):
    name = "flash_attn_varlen_qkvpacked_func"
    _unsupported(name, dropout_p, causal, window_size, softcap, alibi_slopes, return_attn_probs)
    q, k, v = _split(name, qkv, 3, "qkv")
    return _A.varlen(q, k, v, cu_seqlens, cu_seqlens, max_seqlen, max_seqlen, softmax_scale, name)


def flash_attn_varlen_kvpacked_func(q, kv, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p=0.0,
                                    softmax_scale=None, causal=False, window_size=(-1, -1), softcap=0.0,
                                    alibi_slopes=None, deterministic=False, return_attn_probs=False):
    name = "flash_attn_varlen_kvpacked_func"
    _unsupported(name, dropout_p, causal, window_size, softcap, alibi_slopes, return_attn_probs)
    k, v = _split(name, kv, 2, "kv")
    return _A.varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, softmax_scale, name)


def flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, dropout_p=0.0,
                           softmax_scale=None, causal=False, window_size=(-1, -1), softcap=0.0, alibi_slopes=None,
                           deterministic=False, return_attn_probs=False, block_table=None):
    name = "flash_attn_varlen_func"
    _unsupported(name, dropout_p, causal, window_size, softcap, alibi_slopes, return_attn_probs, block_table)
    return _A.varlen(q, k, v, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, softmax_scale, name)


def flash_attn_qkvpacked_func(qkv, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1), softcap=0.0,
                              alibi_slopes=None, deterministic=False, return_attn_probs=False):
    name = "flash_attn_qkvpacked_func"
    _unsupported(name, dropout_p, causal, window_size, softcap, alibi_slopes, return_attn_probs)
    q, k, v = _split(name, qkv, 3, "qkv")
    return _A.dense(q, k, v, softmax_scale, name)


def flash_attn_kvpacked_func(q, kv, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1), softcap=0.0,
                             alibi_slopes=None, deterministic=False, return_attn_probs=False):
    name = "flash_attn_kvpacked_func"
    _unsupported(name, dropout_p, causal, window_size, softcap, alibi_slopes, return_attn_probs)
    k, v = _split(name, kv, 2, "kv")
    return _A.dense(q, k, v, softmax_scale, name)


def flash_attn_func(q, k, v, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1), softcap=0.0,
                    alibi_slopes=None, deterministic=False, return_attn_probs=False):
    name = "flash_attn_func"
    _unsupported(name, dropout_p, causal, window_size, softcap, alibi_slopes, return_attn_probs)
    return _A.dense(q, k, v, softmax_scale, name)
