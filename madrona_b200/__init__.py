"""madrona_b200 -- H100-native drop-in for the Madrona GPU backend.

The product is libmadrona_b200.so (C ABI in include/madrona_b200.h, hand-written
sm_90a CUDA).  This package is the Python-side mirror of the reference's
executor interface (madrona::MWCudaExecutor, include/madrona/mw_gpu.hpp:98-164);
it binds the C ABI with ctypes and exposes exported ECS columns as zero-copy
torch tensors.  There is no CPU fallback: importing works anywhere, but
creating an executor requires the CUDA library and an H100.
"""
from .executor import (  # noqa: F401
    StateConfig,
    CompileConfig,
    MWCudaExecutor,
    MWCudaLaunchGraph,
    MadronaB200Error,
    load_library,
    library_path,
    precompile,
    MeshBVHData,
    MaterialData,
    RigidBodyAssets,
    Navmesh,
    PeerGather,
    Snapshot,
)
from .tensor import (  # noqa: F401
    Tensor, TensorElementType, NamedTensor, TrainInterface, TrainStepInputInterface,
    TrainStepOutputInterface, TrainCheckpointingInterface,
)
