"""dirtorch.ivf (extension): inverted-file search over k-means lists on the GPU; see dirb200.ivf."""
from dirb200.ivf import IVFIndex  # noqa: F401
