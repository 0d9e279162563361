"""pointnet2_ops.pointnet2_utils: the six operators on the GPU (gs_b200.pointnet2); the nn.Module helpers no caller
in the pack uses raise NotImplementedError."""
from gs_b200.pointnet2 import (BallQuery, FurthestPointSampling, GatherOperation, GroupingOperation, ThreeInterpolate,
                               ThreeNN, ball_query, furthest_point_sample, gather_operation, grouping_operation,
                               three_interpolate, three_nn)

_PROVIDED = ("furthest_point_sample, gather_operation, grouping_operation, ball_query, three_nn and "
             "three_interpolate")


def _not_provided(name):
    def fn(*a, **k):
        raise NotImplementedError(f"pointnet2_ops.pointnet2_utils.{name} is not provided: only {_PROVIDED} run on "
                                  f"the GPU here, and no caller in the pack uses {name}")
    fn.__name__ = name
    return fn


QueryAndGroup = _not_provided("QueryAndGroup")
GroupAll = _not_provided("GroupAll")

__all__ = ["furthest_point_sample", "gather_operation", "grouping_operation", "ball_query", "three_nn",
           "three_interpolate", "FurthestPointSampling", "GatherOperation", "GroupingOperation", "BallQuery", "ThreeNN",
           "ThreeInterpolate", "QueryAndGroup", "GroupAll"]
