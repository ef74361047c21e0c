"""equiformer_b200 - sm_90a edge kernels behind Equiformer's equivariant graph attention."""
from . import o3  # noqa: F401

__version__ = "0.1.0"
