"""Builds the reference's own `custom_rasterizer_kernel` (Hunyuan3D's texture-bake rasterizer) into oracle/_ref/, so
tests and benchmarks can hold gs_b200.custom_rasterizer to the reference's binaries.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python oracle/build_ref.py

Two builds of the same three sources (rasterizer.cpp, grid_neighbor.cpp, rasterizer_gpu.cu), for sm_90a:
  * default: nvcc's default FMA contraction, the binary users of the reference run;
  * nofma:   -fmad=false on the device and -ffp-contract=off on the host: the arithmetic the contract restates.
Each lands in oracle/_ref/custom_rasterizer_<variant>/ as custom_rasterizer_kernel_<variant>.so.  A build is skipped
when its stamp (SHA-256 of the sources, the flags and the torch version) is unchanged: each one takes minutes.
The pack is the one COMFYUI_3D_PACK names or, when it is unset, one in a directory next to this repository (both
under ComfyUI's custom_nodes/, say).  When no pack is found this prints why and returns; it never raises, so build()
cannot fail on it.  Nothing from the reference is copied into the repository: the sources are compiled in place.
"""
import hashlib
import importlib.util
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
KERNEL_DIRS = ("Gen_3D_Modules/Hunyuan3D_2_1/hy3dpaint/custom_rasterizer/lib/custom_rasterizer_kernel",
               "Gen_3D_Modules/Hunyuan3D_V2/hy3dgen/texgen/custom_rasterizer/lib/custom_rasterizer_kernel")
SOURCES = ("rasterizer.cpp", "grid_neighbor.cpp", "rasterizer_gpu.cu")
GENCODE = "-gencode=arch=compute_90a,code=sm_90a"
VARIANTS = {
    "default": {"cflags": ["-O3"], "cuda": ["-O3", GENCODE]},
    "nofma": {"cflags": ["-O3", "-ffp-contract=off"],
              "cuda": ["-O3", GENCODE, "-fmad=false", "-Xcompiler", "-ffp-contract=off"]},
}


def _candidates():
    """ComfyUI-3D-Pack checkouts to look in: $COMFYUI_3D_PACK when set, else the directories next to this repository
    (where ComfyUI's custom_nodes/ keeps the pack beside it)."""
    ref = os.environ.get("COMFYUI_3D_PACK")
    if ref:
        return [ref]
    parent = os.path.dirname(os.path.dirname(HERE))
    try:
        return sorted(e.path for e in os.scandir(parent) if e.is_dir() and e.path != os.path.dirname(HERE))
    except OSError:
        return []


def kernel_dir():
    """The reference's custom_rasterizer_kernel source directory, or None."""
    for ref in _candidates():
        for rel in KERNEL_DIRS:
            d = os.path.join(ref, rel)
            try:
                if all(os.access(os.path.join(d, s), os.R_OK) for s in SOURCES):
                    return d
            except OSError:
                continue
    return None


def so_path(variant):
    d = os.path.join(OUT, f"custom_rasterizer_{variant}")
    return os.path.join(d, f"custom_rasterizer_kernel_{variant}.so")


def load(variant):
    """The built reference module for `variant`, or None when it has not been built.  Importing it needs torch."""
    path = so_path(variant)
    if not os.path.isfile(path):
        return None
    import torch  # noqa: F401  (the extension links against torch's libraries)
    name = f"custom_rasterizer_kernel_{variant}"
    if name in sys.modules:
        return sys.modules[name]
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules[name] = mod
    return mod


def _stamp(src_dir, variant):
    import torch
    h = hashlib.sha256()
    for s in SOURCES + ("rasterizer.h",):
        p = os.path.join(src_dir, s)
        if os.path.isfile(p):
            h.update(s.encode() + b"\0" + open(p, "rb").read())
    h.update(repr(VARIANTS[variant]).encode() + torch.__version__.encode())
    return h.hexdigest()


_CHILD = r"""
import os, sys
from torch.utils import cpp_extension
variant, src_dir, out_dir = sys.argv[1], sys.argv[2], sys.argv[3]
flags = %r[variant]
cpp_extension.load(name="custom_rasterizer_kernel_" + variant,
                   sources=[os.path.join(src_dir, s) for s in %r],
                   extra_cflags=flags["cflags"], extra_cuda_cflags=flags["cuda"],
                   build_directory=out_dir, verbose=False)
"""


def build(variants=tuple(VARIANTS), quiet=False):
    """Builds what is stale; returns {variant: status string}.  Never raises."""
    say = (lambda *a: None) if quiet else (lambda *a: print("[oracle/_ref]", *a, flush=True))
    try:
        src = kernel_dir()
        if src is None:
            say("reference custom_rasterizer_kernel not found (set COMFYUI_3D_PACK to a ComfyUI-3D-Pack checkout, or"
                " place one next to this repository); skipping the reference build")
            return {v: "absent" for v in variants}
        status, procs = {}, {}
        for v in variants:
            out_dir = os.path.dirname(so_path(v))
            os.makedirs(out_dir, exist_ok=True)
            stamp_file = os.path.join(out_dir, "STAMP")
            stamp = _stamp(src, v)
            if os.path.isfile(so_path(v)) and os.path.isfile(stamp_file) and open(stamp_file).read() == stamp:
                status[v] = "up to date"
                continue
            env = dict(os.environ, TORCH_CUDA_ARCH_LIST="9.0a", MAX_JOBS=os.environ.get("MAX_JOBS", "4"))
            say(f"building {v} from {src} (a few minutes)")
            log = open(os.path.join(out_dir, "build.log"), "w")
            procs[v] = (subprocess.Popen([sys.executable, "-c", _CHILD % (VARIANTS, SOURCES), v, src, out_dir],
                                         env=env, stdout=log, stderr=subprocess.STDOUT), stamp_file, stamp, log)
        for v, (p, stamp_file, stamp, log) in procs.items():
            rc = p.wait()
            log.close()
            if rc == 0 and os.path.isfile(so_path(v)):
                with open(stamp_file, "w") as f:
                    f.write(stamp)
                status[v] = "built"
            else:
                status[v] = f"failed (rc={rc}, see {os.path.join(os.path.dirname(so_path(v)), 'build.log')})"
            say(v, status[v])
        return status
    except Exception as e:  # the reference build is optional: report, never fail the caller
        say("reference build skipped:", repr(e))
        return {v: f"error: {e!r}" for v in variants}


if __name__ == "__main__":
    print(build())
