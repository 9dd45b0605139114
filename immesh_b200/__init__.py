"""immesh_b200 -- H100-native (sm_90a CUDA) implementation of the ImMesh per-scan
localization + meshing hot path behind a C ABI (include/immesh_b200.h).

The Python layer is only a ctypes harness for tests and benchmarks; the product is
libimmesh_b200.so (hand-written CUDA kernels + C++ host orchestration).
"""
from .api import Lio, Mesh, LioConfig, MeshConfig, load_library, AVIA, VELODYNE  # noqa: F401

__version__ = "0.1.0"
