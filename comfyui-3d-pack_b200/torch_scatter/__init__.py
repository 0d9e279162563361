"""Import-name shim for torch_scatter 2.1's scatter_sum / scatter_add, scatter_mean and scatter_max, the four functions
the pack calls (FlexiCubes loss.py:58-68, Unique3D mesh_reconstruction/opt.py:137 and remesh.py:218,336,
TriplaneGaussian models/pointclouds/pointnet.py:63,75).  They run on the GPU through gs_b200.scatter, which states
the rules.  Differences from the package: no CPU path; fp32, int32 and int64 src only (fp32 for the mean), int64
index only; fp32 sums are a fixed ascending-position fold and max ties resolve to the smallest position, so results
have the same bits on every run.  With this directory on sys.path, `import torch_scatter` resolves here for the
whole process, shadowing an installed torch_scatter.
"""
from gs_b200.scatter import scatter_add, scatter_max, scatter_mean, scatter_sum

__version__ = "2.1.2"

_PROVIDED = "scatter_sum, scatter_add, scatter_mean and scatter_max"


def _not_provided(name):
    def fn(*a, **k):
        raise NotImplementedError(f"torch_scatter.{name} is not provided: only {_PROVIDED} run on the GPU here, "
                                  f"and no caller in the pack uses {name}")
    fn.__name__ = name
    return fn


scatter = _not_provided("scatter")
scatter_mul = _not_provided("scatter_mul")
scatter_min = _not_provided("scatter_min")
scatter_std = _not_provided("scatter_std")
scatter_logsumexp = _not_provided("scatter_logsumexp")
scatter_softmax = _not_provided("scatter_softmax")
scatter_log_softmax = _not_provided("scatter_log_softmax")
segment_csr = _not_provided("segment_csr")
segment_sum_csr = _not_provided("segment_sum_csr")
segment_add_csr = _not_provided("segment_add_csr")
segment_mean_csr = _not_provided("segment_mean_csr")
segment_min_csr = _not_provided("segment_min_csr")
segment_max_csr = _not_provided("segment_max_csr")
gather_csr = _not_provided("gather_csr")
segment_coo = _not_provided("segment_coo")
segment_sum_coo = _not_provided("segment_sum_coo")
segment_add_coo = _not_provided("segment_add_coo")
segment_mean_coo = _not_provided("segment_mean_coo")
segment_min_coo = _not_provided("segment_min_coo")
segment_max_coo = _not_provided("segment_max_coo")
gather_coo = _not_provided("gather_coo")

__all__ = ["scatter_sum", "scatter_add", "scatter_mean", "scatter_max", "scatter", "scatter_mul", "scatter_min",
           "scatter_std", "scatter_logsumexp", "scatter_softmax", "scatter_log_softmax", "segment_csr",
           "segment_sum_csr", "segment_add_csr", "segment_mean_csr", "segment_min_csr", "segment_max_csr", "gather_csr",
           "segment_coo", "segment_sum_coo", "segment_add_coo", "segment_mean_coo", "segment_min_coo",
           "segment_max_coo", "gather_coo", "__version__"]
