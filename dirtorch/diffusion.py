"""dirtorch.diffusion (extension): diffusion re-ranking over the mutual-kNN graph of the database, on CUDA kernels;
see dirb200.diffusion."""
from dirb200.diffusion import DEFAULTS, Diffusion, Graph, check_params, graph_from_knn  # noqa: F401
