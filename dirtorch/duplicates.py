"""dirtorch.duplicates (extension): exact near-duplicate detection and set overlap by range search on the GPU; see
dirb200.duplicates."""
from dirb200.duplicates import Duplicates, near_duplicates, overlap  # noqa: F401
