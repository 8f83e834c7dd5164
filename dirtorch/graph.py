"""dirtorch.graph (extension): graph search over a pruned kNN graph on the GPU; see dirb200.graph."""
from dirb200.graph import GraphIndex  # noqa: F401
