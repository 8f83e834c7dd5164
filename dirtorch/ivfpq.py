"""dirtorch.ivfpq (extension): IVF-PQ search with exact re-ranking on the GPU; see dirb200.ivfpq."""
from dirb200.ivfpq import IVFPQIndex  # noqa: F401
