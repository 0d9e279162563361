"""pointnet2_ops.pointnet2_modules: not provided.  No caller in the pack builds these modules; each name raises
NotImplementedError when called."""


def _not_provided(name):
    def fn(*a, **k):
        raise NotImplementedError(f"pointnet2_ops.pointnet2_modules.{name} is not provided: only the "
                                  "pointnet2_utils operators run on the GPU here, and no caller in the pack uses it")
    fn.__name__ = name
    return fn


PointnetSAModuleMSG = _not_provided("PointnetSAModuleMSG")
PointnetSAModule = _not_provided("PointnetSAModule")
PointnetFPModule = _not_provided("PointnetFPModule")

__all__ = ["PointnetSAModuleMSG", "PointnetSAModule", "PointnetFPModule"]
