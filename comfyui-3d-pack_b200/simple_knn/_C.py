"""`distCUDA2(points[N,3] cuda) -> [N]` mean squared distance to the 3 nearest neighbours, H100-native."""
from gs_b200.rasterizer import knn_mean_dist2 as distCUDA2  # noqa: F401
