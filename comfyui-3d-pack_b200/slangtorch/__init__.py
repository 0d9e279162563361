"""Import-name shim for `slangtorch`, which StableFast3D's TextureBaker (sf3d/texture_baker.py:13) uses to JIT-compile
texture_baker.slang at first use: that needs the Slang compiler and a host toolchain.  Here loadModule serves that one
file, recognised by its SHA-256 (line endings normalised), from prebuilt sm_90a kernels (gs_b200.uv_bake) whose
outputs are bit-identical to the reference's generated CUDA.  Any other Slang file raises NotImplementedError: nothing
is compiled at run time.  With this directory on sys.path, sf3d/texture_baker.py runs unmodified.

The module's bake_uv(uv=, indices=, output=) and interpolate(attr=, indices=, rast=, output=) return a call whose
launchRaw(blockSize=, gridSize=) does the work on the current stream.  As in the reference, thread (x, y) of the launch
handles texel [x, y] (row x, column y), so exactly rows = gridSize[0] * blockSize[0] and cols = gridSize[1] *
blockSize[1] texels are written, clipped to the texture; TextureBaker's res // 16 blocks of 16 leave the last res % 16
rows and columns as the caller allocated them.
"""
import hashlib
import os

from gs_b200 import uv_bake as _uv_bake

# sf3d/texture_baker.slang of StableFast3D (ComfyUI-3D-Pack's Gen_3D_Modules/StableFast3D), "\r\n" read as "\n"
TEXTURE_BAKER_SHA256 = "2368dd0bfa39ceb02398ebfc1101cc2f249e4c78d2dcc576c6835f3525c54fbd"


def file_sha256(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read().replace(b"\r\n", b"\n")).hexdigest()


def _region(blockSize, gridSize):
    b, g = tuple(int(x) for x in blockSize), tuple(int(x) for x in gridSize)
    if len(b) != 3 or len(g) != 3 or min(b + g) < 0:
        raise ValueError(f"blockSize and gridSize must be three non-negative ints, got {blockSize} and {gridSize}")
    if min(b[2], g[2]) == 0:
        return 0, 0
    return g[0] * b[0], g[1] * b[1]


class _Launch:
    def __init__(self, fn, args):
        self._fn, self._args = fn, args

    def launchRaw(self, blockSize, gridSize):
        rows, cols = _region(blockSize, gridSize)
        self._fn(*self._args, rows, cols)


class TextureBakerModule:
    """texture_baker.slang's two kernels."""

    @staticmethod
    def bake_uv(uv, indices, output):
        return _Launch(_uv_bake.rasterize_into, (uv, indices, output))

    @staticmethod
    def interpolate(attr, indices, rast, output):
        return _Launch(lambda a, i, r, o, rows, cols: _uv_bake.interpolate_into(a, r, i, o, rows, cols),
                       (attr, indices, rast, output))


def loadModule(fileName, **kwargs):
    """The module of texture_baker.slang; NotImplementedError for any other file (no Slang compiler here)."""
    path = os.fspath(fileName)
    try:
        digest = file_sha256(path)
    except OSError as e:
        raise NotImplementedError(f"slangtorch.loadModule({path!r}): cannot read the file ({e}); only StableFast3D's "
                                  "texture_baker.slang is provided, prebuilt") from e
    if digest != TEXTURE_BAKER_SHA256:
        raise NotImplementedError(f"slangtorch.loadModule({path!r}): only StableFast3D's texture_baker.slang is "
                                  f"provided, prebuilt; this file (sha256 {digest[:16]}...) would need the Slang "
                                  "compiler")
    return TextureBakerModule()


__all__ = ["loadModule", "TextureBakerModule", "TEXTURE_BAKER_SHA256", "file_sha256"]
