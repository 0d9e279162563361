"""Import-name shim: `import nvdiffrast.torch as dr` (diff_mesh_renderer.py:8, flexicubes_renderer.py:5,
FlexiCubes/util.py:10, mesh_utils.py) resolves to the H100-native mesh ops."""
__version__ = "0.3.3+b200"
