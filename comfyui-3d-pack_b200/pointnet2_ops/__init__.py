"""Import-name shim for pointnet2_ops 3.0's six point-cloud operators, which TriplaneGaussian's snowflake decoder
imports from pointnet2_ops.pointnet2_utils (models/snowflake/utils.py:9): furthest_point_sample, gather_operation,
grouping_operation, ball_query, three_nn and three_interpolate.  They run on the GPU through gs_b200.pointnet2, which
states the rules.  Differences from the package: no CPU path; ties go to the smallest index whatever the launch shape;
an index outside the feature range reads 0 and gets no gradient; gradients have the same bits on every run; and
three_interpolate returns no gradient for `weight` (the package returns zeros).  QueryAndGroup, GroupAll and the
pointnet2_modules classes raise NotImplementedError.  With this directory on sys.path, `import pointnet2_ops` resolves
here for the whole process, shadowing an installed pointnet2_ops.
"""
from . import pointnet2_utils  # noqa: F401

__version__ = "3.0.0"
