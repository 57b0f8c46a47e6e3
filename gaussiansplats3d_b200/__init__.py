"""gaussiansplats3d_b200 -- H100 (sm_90a) depth -> sort -> rasterise engine behind the GaussianSplats3D
sort-worker / SplatMesh boundary.  Compute lives in csrc/libgsplat_b200.so (hand-written CUDA, C ABI in
include/gsplat_b200.h); this package is the host-side mirror of the reference's interface for that path."""
from . import _native
from ._native import GsError
from .engine import Engine, Eye, Uniforms, View, sort_indexes

__all__ = ["Engine", "Eye", "Uniforms", "View", "sort_indexes", "GsError", "_native"]
__version__ = "0.1.0"
