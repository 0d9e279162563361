"""Import-name shim for the part of spconv 2.x that TRELLIS and Stable3DGen use: `spconv.pytorch.SubMConv3d` (kernel
size 1 or 3, stride 1, dilation 1) and `SparseConvTensor` as its container (trellis/modules/sparse/basic.py and
conv/conv_spconv.py).  The convolution runs on the GPU through gs_b200.spconv, which states the rules.  Differences
from the package: no CPU path; duplicate coordinates resolve to their smallest row; every output and gradient has the
same bits on every run; `algo` is accepted and ignored.  Strided or padded SparseConv3d, SparseInverseConv3d,
dilation other than 1 and kernel sizes other than 1 and 3 raise NotImplementedError.  With this directory on
sys.path, `import spconv` resolves here for the whole process, shadowing an installed spconv.
"""
from . import pytorch  # noqa: F401

__version__ = "2.3.6"
