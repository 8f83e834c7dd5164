"""dirtorch.cluster (extension): exact spherical k-means of descriptor collections on the GPU; see dirb200.cluster."""
from dirb200.cluster import SphericalKMeans  # noqa: F401
