"""Import-name shim: `from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer`
(MVs_Algorithms/GaussianSplatting/main_3DGS_renderer.py:840-843) resolves to the H100-native implementation
when `comfyui-3d-pack_b200/` is on sys.path (the reference injects its own paths the same way, __init__.py:12-14)."""
from gs_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians  # noqa: F401
