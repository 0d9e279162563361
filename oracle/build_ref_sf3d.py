"""Builds the reference's own StableFast3D texture baker into oracle/_ref/, so tests and benchmarks can hold
gs_b200.uv_bake to the reference's binaries.

    COMFYUI_3D_PACK=/path/to/ComfyUI-3D-Pack python oracle/build_ref_sf3d.py

The pack ships the CUDA that slangtorch generated from sf3d/texture_baker.slang
(sf3d/.slangtorch_cache/texture_baker/<hash>/texture_baker_cuda.cu).  build() compiles it in place through
oracle/sf3d_ref_launch.cu, which #includes it via -I, with nvcc's default flags for sm_90a, into
oracle/_ref/sf3d_texture_baker/libsf3d_texture_baker_ref.so (seconds).  It rebuilds only when its stamp (SHA-256 of
the two sources and the flags) changes.  The pack is found as oracle/build_ref.py finds it (COMFYUI_3D_PACK, or a
checkout next to this repository); when there is none this prints why and returns.  It never raises, so build()
cannot fail on it.  Nothing from the reference is copied into the repository.  load() opens the library with ctypes.
"""
import ctypes
import glob
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
if os.path.dirname(HERE) not in sys.path:
    sys.path.insert(0, os.path.dirname(HERE))

from oracle.build_ref import GENCODE, OUT, _candidates  # noqa: E402

CACHE_GLOB = "Gen_3D_Modules/StableFast3D/sf3d/.slangtorch_cache/texture_baker/*/texture_baker_cuda.cu"
LAUNCHER = os.path.join(HERE, "sf3d_ref_launch.cu")
OUT_DIR = os.path.join(OUT, "sf3d_texture_baker")
SO = os.path.join(OUT_DIR, "libsf3d_texture_baker_ref.so")
FLAGS = [GENCODE, "-shared", "-Xcompiler", "-fPIC"]     # nvcc's defaults otherwise: FMA contraction, IEEE division


def source():
    """The reference's generated texture_baker_cuda.cu, or None."""
    for ref in _candidates():
        try:
            hits = sorted(glob.glob(os.path.join(ref, CACHE_GLOB)))
        except OSError:
            continue
        for h in hits:
            if os.access(h, os.R_OK):
                return h
    return None


def _nvcc():
    cuda = os.environ.get("CUDA_HOME") or "/usr/local/cuda"
    p = os.path.join(cuda, "bin", "nvcc")
    return p if os.path.isfile(p) else "nvcc"


def build(quiet=False):
    """Builds the SF3D reference baker when stale; returns a status string.  Never raises."""
    say = (lambda *a: None) if quiet else (lambda *a: print("[oracle/_ref]", *a, flush=True))
    try:
        src = source()
        if src is None:
            say("reference SF3D texture_baker_cuda.cu not found (set COMFYUI_3D_PACK to a ComfyUI-3D-Pack checkout, or"
                " place one next to this repository); skipping the SF3D reference build")
            return "absent"
        os.makedirs(OUT_DIR, exist_ok=True)
        h = hashlib.sha256()
        for p in (src, LAUNCHER):
            h.update(open(p, "rb").read() + b"\0")
        h.update(repr(FLAGS).encode())
        stamp, stamp_file = h.hexdigest(), os.path.join(OUT_DIR, "STAMP")
        if os.path.isfile(SO) and os.path.isfile(stamp_file) and open(stamp_file).read() == stamp:
            return "up to date"
        say(f"building the SF3D texture baker from {src}")
        cmd = [_nvcc(), *FLAGS, "-I", os.path.dirname(src), "-o", SO, LAUNCHER]
        with open(os.path.join(OUT_DIR, "build.log"), "w") as log:
            rc = subprocess.run(cmd, stdout=log, stderr=subprocess.STDOUT).returncode
        if rc == 0 and os.path.isfile(SO):
            with open(stamp_file, "w") as f:
                f.write(stamp)
            status = "built"
        else:
            status = f"failed (rc={rc}, see {os.path.join(OUT_DIR, 'build.log')})"
        say("sf3d_texture_baker", status)
        return status
    except Exception as e:  # the reference build is optional: report, never fail the caller
        say("SF3D reference build skipped:", repr(e))
        return f"error: {e!r}"


def load():
    """ctypes handle of the built SF3D reference baker, or None.  sf3d_ref_bake_uv(uv, V, indices, F, out, H, W, bx, by,
    gx, gy, stream) and sf3d_ref_interpolate(attr, V, indices, F, rast, out, H, W, bx, by, gx, gy, stream) launch the
    reference kernels with launchRaw's block and grid; both return a cudaError_t."""
    if not os.path.isfile(SO):
        return None
    lib = ctypes.CDLL(SO)
    P, I, Un = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint
    lib.sf3d_ref_bake_uv.restype = I
    lib.sf3d_ref_bake_uv.argtypes = [P, I, P, I, P, I, I, Un, Un, Un, Un, P]
    lib.sf3d_ref_interpolate.restype = I
    lib.sf3d_ref_interpolate.argtypes = [P, I, P, I, P, P, I, I, Un, Un, Un, Un, P]
    return lib


if __name__ == "__main__":
    print(build())
