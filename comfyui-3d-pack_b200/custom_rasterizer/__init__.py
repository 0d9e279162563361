"""Import-name shim for Hunyuan3D's `custom_rasterizer` package (render.py's rasterize / interpolate), which the 2.0
(texgen/differentiable_renderer/mesh_render.py:145) and 2.1 (hy3dpaint/DifferentiableRenderer/MeshRender.py:373)
texture pipelines import for every render and bake.  It runs on the GPU through gs_b200.custom_rasterizer, whose
findices and barycentrics are bit-identical to the package's CPU path.  No CPU path.  The mesh loaders the 2.0
package re-exports from io_glb / io_obj are not provided and raise NotImplementedError.  With this directory on
sys.path, `import custom_rasterizer` resolves here for the whole process, shadowing an installed wheel.
"""
from gs_b200.custom_rasterizer import interpolate, rasterize

_LOADERS = ("get_buffer_data", "get_attribute_data", "get_image_data", "convert_triangle_strip_to_triangles",
            "convert_triangle_fan_to_triangles", "get_node_transform", "get_world_transform", "LoadGlb",
            "RotatePrimitives", "LoadObj", "LoadObjWithTexture")


def _not_provided(name):
    def fn(*args, **kwargs):
        raise NotImplementedError(f"custom_rasterizer.{name} (a mesh loader of the package's io_glb / io_obj) is not "
                                  "provided: the pack's pipelines load meshes elsewhere")
    fn.__name__ = name
    return fn


globals().update({n: _not_provided(n) for n in _LOADERS})

__all__ = ["rasterize", "interpolate", *_LOADERS]
