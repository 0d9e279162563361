"""gs_b200 — H100-native (sm_90a) Gaussian-splatting rasterizer, host side.

Python is the reference's host language for this path; this package mirrors the
`diff_gaussian_rasterization` interface over the C ABI in include/gs_b200.h.
"""
from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians  # noqa: F401
