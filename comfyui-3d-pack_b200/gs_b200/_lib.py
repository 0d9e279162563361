"""ctypes binding of the C ABI declared in include/*.h.

Every function the headers declare is bound at import with the restype / argtypes its prototype gives, and every
integer `#define GS_B200_<NAME>` and `enum { GS_B200_<NAME> = n }` becomes the module attribute `<NAME>`, so the
headers are the only place a signature or constant is written.

The CUDA library is the product; there is NO CPU fallback: importing this module
raises if ``libgs_b200.so`` has not been built (``python __graft_entry__.py`` or
``csrc/build.sh``).
"""
import ctypes as C
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgs_b200.so")
_INCLUDE = os.path.join(os.path.dirname(os.path.dirname(_HERE)), "include")


class View(C.Structure):
    _fields_ = [("image_height", C.c_int32), ("image_width", C.c_int32), ("tanfovx", C.c_float),
                ("tanfovy", C.c_float), ("bg", C.c_void_p), ("scale_modifier", C.c_float),
                ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("sh_degree", C.c_int32),
                ("campos", C.c_void_p), ("prefiltered", C.c_int32), ("debug", C.c_int32)]


class State(C.Structure):
    _fields_ = [("geom", C.c_void_p), ("point_list", C.c_void_p), ("tile_keys", C.c_void_p),
                ("ranges", C.c_void_p), ("n_contrib", C.c_void_p), ("final_T", C.c_void_p),
                ("num_rendered", C.c_int64), ("num_gaussians", C.c_int32), ("tiles_x", C.c_int32),
                ("tiles_y", C.c_int32), ("owned", C.c_void_p * 4)]


ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_int32, C.c_size_t)
VIEW_HOOK = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_int32, C.c_void_p)
GRAD_SINK = C.CFUNCTYPE(None, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p)

STAGE_NAMES = ["preprocess", "depth_sort", "scan", "emit", "tile_sort", "ranges", "composite_fwd",
               "composite_bwd", "preprocess_bwd"]

# C type (`const` dropped, `*` attached) -> ctypes type.  Any other pointer is c_void_p; any other type is refused.
_CTYPES = {"int32_t": C.c_int32, "int64_t": C.c_int64, "float": C.c_float, "double": C.c_double, "size_t": C.c_size_t,
           "gs_b200_view*": C.POINTER(View), "gs_b200_state*": C.POINTER(State), "gs_b200_alloc_fn": ALLOC_FN,
           "gs_b200_view_hook": VIEW_HOOK, "gs_b200_grad_sink": GRAD_SINK}
_RESTYPES = {**_CTYPES, "void": None, "char*": C.c_char_p}
_PROTO = re.compile(r"(\w[\w\s]*?\**)\s*\b((?:gs|dr|ngp)_b200_\w+)\s*\(([^()]*)\)\s*;")


def _ctype(decl, fn, table=_CTYPES):
    t = re.sub(r"\s*\*\s*", "*", " ".join(re.sub(r"\bconst\b", " ", decl).split()))
    if t in table:
        return table[t]
    if t.endswith("*"):
        return C.c_void_p
    raise ImportError(f"{fn}: C type '{t}' has no ctypes mapping in gs_b200/_lib.py")


def prototypes(src):
    """{name: (restype, argtypes)} of every gs/dr/ngp_b200_* function declared in the header text `src`."""
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"^\s*#.*$", "", src, flags=re.M)
    out = {}
    for ret, name, params in _PROTO.findall(src):
        if ret.split()[0] == "typedef":
            continue
        params = [p for p in params.split(",") if p.strip() not in ("", "void")]
        out[name] = (_ctype(ret, name, _RESTYPES), [_ctype(re.sub(r"\w+\s*$", "", p), name) for p in params])
    return out


def constants(src):
    """{NAME: value} of the integer `#define GS_B200_<NAME> n` and `enum { GS_B200_<NAME> = n }` in header `src`."""
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    found = re.findall(r"^[ \t]*#[ \t]*define[ \t]+GS_B200_(\w+)[ \t]+(\d+)[ \t]*$", src, flags=re.M)
    found += re.findall(r"\bGS_B200_(\w+)\s*=\s*(\d+)", src)
    return {k: int(v) for k, v in found}


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: the sm_90a CUDA library has not been built. "
        "Run `python __graft_entry__.py` (or comfyui-3d-pack_b200/csrc/build.sh). There is no CPU fallback.")

lib = C.CDLL(LIB_PATH)


def _bind():
    if not os.path.isdir(_INCLUDE):
        raise ImportError(f"{_INCLUDE} is missing: gs_b200 binds its library from the headers there.")
    for h in sorted(f for f in os.listdir(_INCLUDE) if f.endswith(".h")):
        with open(os.path.join(_INCLUDE, h)) as f:
            src = f.read()
        for name, (restype, argtypes) in prototypes(src).items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
        globals().update(constants(src))


_bind()


def last_error() -> str:
    return lib.gs_b200_last_error().decode("utf-8", "replace")


def check(rc: int):
    if rc != 0:
        raise RuntimeError(f"gs_b200: {last_error()}")


def stream():
    """The current torch CUDA stream, as the `void* stream` every entry point takes."""
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    """A tensor's device address; NULL for None or an empty tensor."""
    return C.c_void_p(t.data_ptr() if t is not None and t.numel() else None)
