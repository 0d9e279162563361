"""Import-name shim for `custom_rasterizer_kernel`, the compiled module under Hunyuan3D's custom_rasterizer package.
`rasterize_image` runs on the GPU through gs_b200.custom_rasterizer, so the package's own render.py runs unchanged over
it.  `build_hierarchy` and `build_hierarchy_with_feat` raise NotImplementedError: nothing in the pack calls them.
No CPU path: CPU tensors raise RuntimeError.
"""
from gs_b200.custom_rasterizer import build_hierarchy, build_hierarchy_with_feat, rasterize_image

__all__ = ["rasterize_image", "build_hierarchy", "build_hierarchy_with_feat"]
