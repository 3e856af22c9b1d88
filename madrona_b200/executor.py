"""ctypes binding of include/madrona_b200.h.

Names and argument meaning follow the reference's host API
(include/madrona/mw_gpu.hpp): StateConfig / CompileConfig fields are the same,
MWCudaExecutor has buildLaunchGraph / buildLaunchGraphAllTaskGraphs / run /
runAsync / getExported.  Errors that the reference turns into FATAL() (abort)
are raised as MadronaB200Error here.
"""
from __future__ import annotations

import ctypes
import os
import weakref
from dataclasses import dataclass, field
from typing import Optional, Sequence

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
_LIB = None

EXPORTED_SYMBOLS = [
    "mb2_init_cuda",
    "mb2_executor_create",
    "mb2_executor_destroy",
    "mb2_build_launch_graph",
    "mb2_build_launch_graph_all",
    "mb2_build_render_graph",
    "mb2_launch_graph_destroy",
    "mb2_run",
    "mb2_run_async",
    "mb2_get_exported",
    "mb2_last_error",
    "mb2_get_exported_num_rows",
    "mb2_get_exported_row_bytes",
    "mb2_launch_graph_num_kernels",
    "mb2_launch_graph_num_branches",
    "mb2_executor_stream",
    "mb2_jit_precompile",
    "mb2_profile_nodes",
    "mb2_version",
    "mb2_init_cuda_ctx",
    "mb2_device_of_context",
    "mb2_build_mesh_bvhs",
    "mb2_mesh_bvh_data_view",
    "mb2_mesh_bvh_triangle_sources",
    "mb2_mesh_bvh_data_destroy",
    "mb2_init_material_data",
    "mb2_material_data_view",
    "mb2_material_data_destroy",
    "mb2_process_rigid_body_assets",
    "mb2_object_manager_ptr",
    "mb2_object_manager_host_assets",
    "mb2_object_manager_destroy",
    "mb2_navmesh_create",
    "mb2_navmesh_view",
    "mb2_navmesh_host_arrays",
    "mb2_navmesh_destroy",
    "mb2_render_debug_hits",
    "mb2_render_debug_buffer",
    "mb2_peer_gather_create",
    "mb2_peer_gather_local_handle",
    "mb2_peer_gather_connect",
    "mb2_peer_gather_push_async",
    "mb2_peer_gather_wait_async",
    "mb2_peer_gather_release_async",
    "mb2_peer_gather_buffer",
    "mb2_peer_gather_destroy",
    "mb2_snapshot_create",
    "mb2_snapshot_save",
    "mb2_snapshot_restore",
    "mb2_snapshot_bytes",
    "mb2_snapshot_saved_bytes",
    "mb2_snapshot_destroy",
]


class MadronaB200Error(RuntimeError):
    pass


class _StateConfigC(ctypes.Structure):
    _fields_ = [
        ("world_init_ptr", ctypes.c_void_p),
        ("num_world_init_bytes", ctypes.c_uint32),
        ("user_config_ptr", ctypes.c_void_p),
        ("num_user_config_bytes", ctypes.c_uint32),
        ("num_world_data_bytes", ctypes.c_uint32),
        ("world_data_alignment", ctypes.c_uint32),
        ("num_worlds", ctypes.c_uint32),
        ("num_taskgraphs", ctypes.c_uint32),
        ("num_exported_buffers", ctypes.c_uint32),
    ]


class _CompileConfigC(ctypes.Structure):
    _fields_ = [
        ("user_sources", ctypes.POINTER(ctypes.c_char_p)),
        ("num_user_sources", ctypes.c_uint32),
        ("user_compile_flags", ctypes.POINTER(ctypes.c_char_p)),
        ("num_user_compile_flags", ctypes.c_uint32),
        ("opt_mode", ctypes.c_uint32),
    ]


class _MeshBVHViewC(ctypes.Structure):       # == render::MeshBVHData
    _fields_ = [
        ("nodes", ctypes.c_void_p), ("num_nodes", ctypes.c_uint64),
        ("leaf_material", ctypes.c_void_p), ("num_leaves", ctypes.c_uint64),
        ("vertices", ctypes.c_void_p), ("num_verts", ctypes.c_uint64),
        ("mesh_bvhs", ctypes.c_void_p), ("num_bvhs", ctypes.c_uint64),
    ]


class _MaterialViewC(ctypes.Structure):      # == render::MaterialData
    _fields_ = [
        ("textures", ctypes.c_void_p), ("num_texture_buffers", ctypes.c_uint32),
        ("texture_buffers", ctypes.c_void_p), ("materials", ctypes.c_void_p),
    ]


class _RenderConfigC(ctypes.Structure):      # == madrona::CudaBatchRenderConfig + image size
    _fields_ = [
        ("render_mode", ctypes.c_uint32),
        ("geo_bvh_data", _MeshBVHViewC),
        ("material_data", _MaterialViewC),
        ("render_resolution", ctypes.c_uint32),
        ("near_plane", ctypes.c_float),
        ("far_plane", ctypes.c_float),
        # non-square images: both nonzero, render_resolution 0 (or equal to both)
        ("render_width", ctypes.c_uint32),
        ("render_height", ctypes.c_uint32),
    ]


class _SourceHullC(ctypes.Structure):
    _fields_ = [("positions", ctypes.c_void_p), ("num_vertices", ctypes.c_uint32),
                ("indices", ctypes.c_void_p), ("face_counts", ctypes.c_void_p),
                ("num_faces", ctypes.c_uint32)]


class _SourcePrimC(ctypes.Structure):
    _fields_ = [("type", ctypes.c_uint32), ("sphere_radius", ctypes.c_float), ("hull_idx", ctypes.c_uint32)]


class _SourceObjectC(ctypes.Structure):
    _fields_ = [("prims", ctypes.POINTER(_SourcePrimC)), ("num_prims", ctypes.c_uint32),
                ("inv_mass", ctypes.c_float), ("mu_s", ctypes.c_float), ("mu_d", ctypes.c_float)]


class _RigidBodyAssetsC(ctypes.Structure):
    _fields_ = [("half_edges", ctypes.c_void_p), ("face_base_half_edges", ctypes.c_void_p),
                ("face_planes", ctypes.c_void_p), ("vertices", ctypes.c_void_p),
                ("num_half_edges", ctypes.c_uint32), ("num_faces", ctypes.c_uint32),
                ("num_verts", ctypes.c_uint32),
                ("primitives", ctypes.c_void_p), ("primitive_aabbs", ctypes.c_void_p),
                ("metadatas", ctypes.c_void_p), ("obj_aabbs", ctypes.c_void_p),
                ("prim_offsets", ctypes.c_void_p), ("prim_counts", ctypes.c_void_p),
                ("num_convex_hulls", ctypes.c_uint32), ("total_num_primitives", ctypes.c_uint32),
                ("num_objs", ctypes.c_uint32)]


class _NavmeshArraysC(ctypes.Structure):   # == mb2_navmesh_arrays
    _fields_ = [("vertices", ctypes.c_void_p), ("tri_indices", ctypes.c_void_p),
                ("tri_adjacency", ctypes.c_void_p), ("alias_table", ctypes.c_void_p),
                ("num_verts", ctypes.c_uint32), ("num_tris", ctypes.c_uint32)]


class _MeshSourceC(ctypes.Structure):
    _fields_ = [
        ("positions", ctypes.c_void_p), ("uvs", ctypes.c_void_p), ("num_vertices", ctypes.c_uint32),
        ("indices", ctypes.c_void_p), ("num_triangles", ctypes.c_uint32), ("material_idx", ctypes.c_int32),
    ]


class _SourceTextureC(ctypes.Structure):    # == imp::SourceTexture
    _fields_ = [("data", ctypes.c_void_p), ("format", ctypes.c_int32), ("width", ctypes.c_uint32),
                ("height", ctypes.c_uint32), ("num_bytes", ctypes.c_uint64)]


class _SourceMaterialC(ctypes.Structure):   # == imp::SourceMaterial
    _fields_ = [("color", ctypes.c_float * 4), ("texture_idx", ctypes.c_int32),
                ("roughness", ctypes.c_float), ("metalness", ctypes.c_float)]


def library_path() -> str:
    # MADRONA_B200_LIB: an alternative build of the same library (A/B measurements)
    return os.environ.get("MADRONA_B200_LIB") or os.path.join(_PKG_DIR, "libmadrona_b200.so")


def load_library() -> ctypes.CDLL:
    """Load libmadrona_b200.so; fails loudly if it has not been built."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = library_path()
    if not os.path.exists(path):
        raise MadronaB200Error(
            f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C madrona_b200`). There is no CPU fallback.")
    lib = ctypes.CDLL(path)
    vp = ctypes.c_void_p
    lib.mb2_init_cuda.argtypes = [ctypes.c_int]
    lib.mb2_init_cuda.restype = ctypes.c_int
    lib.mb2_executor_create.argtypes = [ctypes.POINTER(_StateConfigC),
                                        ctypes.POINTER(_CompileConfigC),
                                        ctypes.c_int, ctypes.POINTER(_RenderConfigC)]
    lib.mb2_executor_create.restype = vp
    lib.mb2_executor_destroy.argtypes = [vp]
    lib.mb2_executor_destroy.restype = None
    lib.mb2_build_launch_graph.argtypes = [vp, ctypes.POINTER(ctypes.c_uint32),
                                           ctypes.c_uint32, ctypes.c_char_p]
    lib.mb2_build_launch_graph.restype = vp
    lib.mb2_build_launch_graph_all.argtypes = [vp]
    lib.mb2_build_launch_graph_all.restype = vp
    lib.mb2_build_render_graph.argtypes = [vp]
    lib.mb2_build_render_graph.restype = vp
    lib.mb2_launch_graph_destroy.argtypes = [vp]
    lib.mb2_launch_graph_destroy.restype = None
    lib.mb2_run.argtypes = [vp, vp]
    lib.mb2_run.restype = ctypes.c_int
    lib.mb2_run_async.argtypes = [vp, vp, vp]
    lib.mb2_run_async.restype = ctypes.c_int
    lib.mb2_get_exported.argtypes = [vp, ctypes.c_int64]
    lib.mb2_get_exported.restype = vp
    lib.mb2_last_error.argtypes = []
    lib.mb2_last_error.restype = ctypes.c_char_p
    lib.mb2_get_exported_num_rows.argtypes = [vp, ctypes.c_int64]
    lib.mb2_get_exported_num_rows.restype = ctypes.c_int64
    lib.mb2_get_exported_row_bytes.argtypes = [vp, ctypes.c_int64]
    lib.mb2_get_exported_row_bytes.restype = ctypes.c_int64
    lib.mb2_launch_graph_num_kernels.argtypes = [vp]
    lib.mb2_launch_graph_num_kernels.restype = ctypes.c_int64
    lib.mb2_launch_graph_num_branches.argtypes = [vp]
    lib.mb2_launch_graph_num_branches.restype = ctypes.c_int64
    lib.mb2_executor_stream.argtypes = [vp]
    lib.mb2_executor_stream.restype = vp
    lib.mb2_jit_precompile.argtypes = [ctypes.POINTER(_CompileConfigC)]
    lib.mb2_jit_precompile.restype = ctypes.c_int
    lib.mb2_profile_nodes.argtypes = [vp, ctypes.POINTER(ctypes.c_uint32), ctypes.c_uint32,
                                      ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint64]
    lib.mb2_profile_nodes.restype = ctypes.c_int64
    lib.mb2_version.argtypes = []
    lib.mb2_version.restype = ctypes.c_char_p
    lib.mb2_build_mesh_bvhs.argtypes = [ctypes.POINTER(_MeshSourceC), ctypes.c_uint32, ctypes.c_int]
    lib.mb2_build_mesh_bvhs.restype = vp
    lib.mb2_mesh_bvh_data_view.argtypes = [vp, ctypes.c_int]
    lib.mb2_mesh_bvh_data_view.restype = ctypes.POINTER(_MeshBVHViewC)
    lib.mb2_mesh_bvh_triangle_sources.argtypes = [vp]
    lib.mb2_mesh_bvh_triangle_sources.restype = ctypes.POINTER(ctypes.c_uint32)
    lib.mb2_mesh_bvh_data_destroy.argtypes = [vp]
    lib.mb2_mesh_bvh_data_destroy.restype = None
    lib.mb2_init_material_data.argtypes = [ctypes.POINTER(_SourceMaterialC), ctypes.c_uint32,
                                           ctypes.POINTER(_SourceTextureC), ctypes.c_uint32, ctypes.c_int]
    lib.mb2_init_material_data.restype = vp
    lib.mb2_material_data_view.argtypes = [vp]
    lib.mb2_material_data_view.restype = ctypes.POINTER(_MaterialViewC)
    lib.mb2_material_data_destroy.argtypes = [vp]
    lib.mb2_material_data_destroy.restype = None
    lib.mb2_process_rigid_body_assets.argtypes = [ctypes.POINTER(_SourceHullC), ctypes.c_uint32,
                                                  ctypes.POINTER(_SourceObjectC), ctypes.c_uint32, ctypes.c_int]
    lib.mb2_process_rigid_body_assets.restype = vp
    lib.mb2_object_manager_ptr.argtypes = [vp, ctypes.c_int]
    lib.mb2_object_manager_ptr.restype = vp
    lib.mb2_object_manager_host_assets.argtypes = [vp, ctypes.POINTER(_RigidBodyAssetsC)]
    lib.mb2_object_manager_host_assets.restype = None
    lib.mb2_object_manager_destroy.argtypes = [vp]
    lib.mb2_object_manager_destroy.restype = None
    lib.mb2_navmesh_create.argtypes = [vp, ctypes.c_uint32, vp, ctypes.c_uint32, vp, vp, ctypes.c_uint32,
                                       ctypes.c_int]
    lib.mb2_navmesh_create.restype = vp
    lib.mb2_navmesh_view.argtypes = [vp]
    lib.mb2_navmesh_view.restype = vp
    lib.mb2_navmesh_host_arrays.argtypes = [vp, ctypes.POINTER(_NavmeshArraysC)]
    lib.mb2_navmesh_host_arrays.restype = None
    lib.mb2_navmesh_destroy.argtypes = [vp]
    lib.mb2_navmesh_destroy.restype = None
    lib.mb2_render_debug_hits.argtypes = [vp]
    lib.mb2_render_debug_hits.restype = vp
    lib.mb2_render_debug_buffer.argtypes = [vp, ctypes.c_int, ctypes.POINTER(ctypes.c_int64)]
    lib.mb2_render_debug_buffer.restype = vp
    lib.mb2_peer_gather_create.argtypes = [vp, ctypes.POINTER(ctypes.c_int64), ctypes.c_uint32,
                                           ctypes.POINTER(ctypes.c_uint64), ctypes.c_uint32, ctypes.c_uint32]
    lib.mb2_peer_gather_create.restype = vp
    lib.mb2_peer_gather_local_handle.argtypes = [vp, ctypes.c_char_p]
    lib.mb2_peer_gather_local_handle.restype = ctypes.c_int
    lib.mb2_peer_gather_connect.argtypes = [vp, ctypes.c_char_p]
    lib.mb2_peer_gather_connect.restype = ctypes.c_int
    for name in ("push", "wait", "release"):
        fn = getattr(lib, f"mb2_peer_gather_{name}_async")
        fn.argtypes = [vp, vp]
        fn.restype = ctypes.c_int
    lib.mb2_peer_gather_buffer.argtypes = [vp, ctypes.c_uint32, ctypes.c_uint32]
    lib.mb2_peer_gather_buffer.restype = vp
    lib.mb2_peer_gather_destroy.argtypes = [vp]
    lib.mb2_peer_gather_destroy.restype = None
    lib.mb2_snapshot_create.argtypes = [vp]
    lib.mb2_snapshot_create.restype = vp
    for name in ("save", "restore"):
        fn = getattr(lib, f"mb2_snapshot_{name}")
        fn.argtypes = [vp, vp, vp]
        fn.restype = ctypes.c_int
    lib.mb2_snapshot_bytes.argtypes = [vp]
    lib.mb2_snapshot_bytes.restype = ctypes.c_int64
    lib.mb2_snapshot_saved_bytes.argtypes = [vp]
    lib.mb2_snapshot_saved_bytes.restype = ctypes.c_int64
    lib.mb2_snapshot_destroy.argtypes = [vp]
    lib.mb2_snapshot_destroy.restype = None
    _LIB = lib
    return lib


def _last_error(lib) -> str:
    msg = lib.mb2_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


@dataclass
class StateConfig:
    """== madrona::StateConfig (mw_gpu.hpp:25-51).  worldInit / userConfig are
    bytes-like host buffers (numpy arrays or bytes)."""
    worldInit: bytes
    numWorldInitBytes: int
    userConfig: bytes
    numWorldDataBytes: int
    worldDataAlignment: int
    numWorlds: int
    numTaskGraphs: int
    numExportedBuffers: int


@dataclass
class CompileConfig:
    """== madrona::CompileConfig (mw_gpu.hpp:53-73)."""
    userSources: Sequence[str]
    userCompileFlags: Sequence[str] = field(default_factory=list)
    optMode: int = 1   # LTO

    def _to_c(self):
        srcs = (ctypes.c_char_p * max(len(self.userSources), 1))(
            *[os.fspath(s).encode() for s in self.userSources])
        flags = (ctypes.c_char_p * max(len(self.userCompileFlags), 1))(
            *[f.encode() for f in self.userCompileFlags])
        c = _CompileConfigC(srcs, len(self.userSources), flags,
                            len(self.userCompileFlags), self.optMode)
        return c, (srcs, flags)


def precompile(compile_cfg: CompileConfig) -> None:
    """JIT the simulator for sm_90a into the in-tree kernel cache (no GPU needed)."""
    lib = load_library()
    c, keep = compile_cfg._to_c()
    if lib.mb2_jit_precompile(ctypes.byref(c)) != 0:
        raise MadronaB200Error(_last_error(lib))
    del keep


def _as_bytes(buf) -> bytes:
    if buf is None:
        return b""
    if isinstance(buf, (bytes, bytearray)):
        return bytes(buf)
    return bytes(memoryview(buf).cast("B"))


class MWCudaLaunchGraph:
    def __init__(self, lib, handle, owner):
        self._lib = lib
        self._h = handle
        self._owner = owner   # keep the executor alive

    @property
    def num_kernels(self) -> int:
        return int(self._lib.mb2_launch_graph_num_kernels(self._h))

    @property
    def num_branches(self) -> int:
        return int(self._lib.mb2_launch_graph_num_branches(self._h))

    def __del__(self):
        try:
            if self._h and self._owner._h:
                self._lib.mb2_launch_graph_destroy(self._h)
        except Exception:
            pass
        self._h = None


class _CudaView:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {
            "shape": tuple(shape), "typestr": typestr,
            "data": (int(ptr), False), "version": 2, "strides": None,
        }


_TYPESTR = {"float32": "<f4", "int32": "<i4", "uint32": "<u4", "uint8": "|u1",
            "int64": "<i8", "float64": "<f8", "int8": "|i1", "int16": "<i2", "uint16": "<u2"}


class MWCudaExecutor:
    """Mirror of madrona::MWCudaExecutor (mw_gpu.hpp:118-164)."""

    @staticmethod
    def initCUDA(gpu_id: int) -> int:
        lib = load_library()
        if lib.mb2_init_cuda(gpu_id) != 0:
            raise MadronaB200Error(_last_error(lib))
        return gpu_id

    def __init__(self, state_cfg: StateConfig, compile_cfg: CompileConfig,
                 gpu_id: int = 0, render_cfg=None):
        self._lib = load_library()
        self._h = None
        self._snapshots = weakref.WeakSet()
        self.gpu_id = gpu_id
        self.num_worlds = state_cfg.numWorlds
        self.num_taskgraphs = state_cfg.numTaskGraphs
        init = _as_bytes(state_cfg.worldInit)
        if len(init) != state_cfg.numWorldInitBytes * state_cfg.numWorlds:
            raise MadronaB200Error("worldInit must hold numWorlds * numWorldInitBytes bytes")
        ucfg = _as_bytes(state_cfg.userConfig)
        init_buf = ctypes.create_string_buffer(init, max(len(init), 1))
        ucfg_buf = ctypes.create_string_buffer(ucfg, max(len(ucfg), 1))
        sc = _StateConfigC(
            ctypes.cast(init_buf, ctypes.c_void_p), state_cfg.numWorldInitBytes,
            ctypes.cast(ucfg_buf, ctypes.c_void_p), len(ucfg),
            state_cfg.numWorldDataBytes, state_cfg.worldDataAlignment,
            state_cfg.numWorlds, state_cfg.numTaskGraphs, state_cfg.numExportedBuffers)
        cc, keep = compile_cfg._to_c()
        rc = ctypes.byref(render_cfg) if render_cfg is not None else None
        h = self._lib.mb2_executor_create(ctypes.byref(sc), ctypes.byref(cc), gpu_id, rc)
        del keep
        if not h:
            raise MadronaB200Error(_last_error(self._lib))
        self._h = h

    # -- reference API ---------------------------------------------------
    def buildLaunchGraph(self, taskgraph_ids, stat_name: Optional[str] = None):
        if isinstance(taskgraph_ids, int):
            taskgraph_ids = [taskgraph_ids]
        ids = (ctypes.c_uint32 * len(taskgraph_ids))(*[int(i) for i in taskgraph_ids])
        g = self._lib.mb2_build_launch_graph(
            self._h, ids, len(taskgraph_ids), stat_name.encode() if stat_name else None)
        if not g:
            raise MadronaB200Error(_last_error(self._lib))
        return MWCudaLaunchGraph(self._lib, g, self)

    def buildLaunchGraphAllTaskGraphs(self):
        g = self._lib.mb2_build_launch_graph_all(self._h)
        if not g:
            raise MadronaB200Error(_last_error(self._lib))
        return MWCudaLaunchGraph(self._lib, g, self)

    def buildRenderGraph(self):
        g = self._lib.mb2_build_render_graph(self._h)
        if not g:
            raise MadronaB200Error(_last_error(self._lib))
        return MWCudaLaunchGraph(self._lib, g, self)

    def run(self, graph: MWCudaLaunchGraph) -> None:
        if self._lib.mb2_run(self._h, graph._h) != 0:
            raise MadronaB200Error(_last_error(self._lib))

    def runAsync(self, graph: MWCudaLaunchGraph, stream) -> None:
        s = getattr(stream, "cuda_stream", stream)
        if self._lib.mb2_run_async(self._h, graph._h, ctypes.c_void_p(int(s))) != 0:
            raise MadronaB200Error(_last_error(self._lib))

    def getExported(self, slot: int) -> int:
        p = self._lib.mb2_get_exported(self._h, int(slot))
        if not p:
            raise MadronaB200Error(f"export slot {slot} is empty")
        return int(p)

    # -- helpers (the role of madrona::py::Tensor, include/madrona/py/utils.hpp:73-141)
    def exportedNumRows(self, slot: int) -> int:
        return int(self._lib.mb2_get_exported_num_rows(self._h, int(slot)))

    def exportedRowBytes(self, slot: int) -> int:
        return int(self._lib.mb2_get_exported_row_bytes(self._h, int(slot)))

    def profileNodes(self, taskgraph_ids=None, reps: int = 10):
        """Per-node device time + algorithmic bytes; advances the sim by `reps` steps."""
        import json
        if taskgraph_ids is None:
            taskgraph_ids = list(range(self.num_taskgraphs))
        ids = (ctypes.c_uint32 * len(taskgraph_ids))(*[int(i) for i in taskgraph_ids])
        buf = ctypes.create_string_buffer(1 << 20)
        n = self._lib.mb2_profile_nodes(self._h, ids, len(taskgraph_ids), reps, buf, len(buf))
        if n < 0:
            raise MadronaB200Error(_last_error(self._lib))
        return json.loads(buf.value.decode())

    @property
    def stream(self) -> int:
        return int(self._lib.mb2_executor_stream(self._h) or 0)

    def tensor(self, slot: int, dtype: str, shape: Sequence[int]):
        """Zero-copy torch view of an exported column on this executor's GPU."""
        import torch
        view = _CudaView(self.getExported(slot), shape, _TYPESTR[dtype])
        return torch.as_tensor(view, device=f"cuda:{self.gpu_id}")

    def exportedTensor(self, slot: int, type, dimensions: Sequence[int]):
        """madrona::py::Tensor over an exported column (what a sim's Manager returns)."""
        from .tensor import Tensor
        return Tensor(self.getExported(slot), type, dimensions, gpu_id=self.gpu_id)

    def renderDebugHits(self, num_views: int, height: int, width: Optional[int] = None):
        """int32 [views, height, width, 2] (instance, triangle) per pixel; width defaults to height
        (square images).  Needs MADRONA_B200_RENDER_DEBUG=1."""
        import torch
        p = self._lib.mb2_render_debug_hits(self._h)
        if not p:
            raise MadronaB200Error("no debug hit buffer (set MADRONA_B200_RENDER_DEBUG=1 before creating the executor)")
        view = _CudaView(p, (num_views, height, height if width is None else width, 2), "<i4")
        return torch.as_tensor(view, device=f"cuda:{self.gpu_id}")

    def renderDebugStructures(self):
        """(tlas_nodes u8 [N, 60], tlas_counts [W], instances u8 [N, 76], instance_counts [W],
        instance_offsets [W]) of the last render-prepare (test hook).  Compact layouts: world w's
        instances and TLAS nodes (node 0 = root) start at instance_offsets[w]; N = visible
        instances of all worlds."""
        import torch
        stride = ctypes.c_int64(0)

        def fetch(which, shape, typestr):
            p = self._lib.mb2_render_debug_buffer(self._h, which, ctypes.byref(stride))
            if not p:
                raise MadronaB200Error("no renderer")
            return torch.as_tensor(_CudaView(p, shape, typestr), device=f"cuda:{self.gpu_id}").cpu().numpy()

        W = self.num_worlds
        ncount, icount, offsets = fetch(2, (W,), "<i4"), fetch(4, (W,), "<i4"), fetch(5, (W,), "<i4")
        total = int(offsets[-1] + icount[-1])
        nodes = fetch(1, (max(total, 1), 60), "|u1")[:total]
        inst = fetch(3, (max(total, 1), 76), "|u1")[:total]
        return nodes, ncount, inst, icount, offsets

    def peerGather(self, slots, shapes, dtypes, world_size: int, rank: int):
        """NVLink peer-store gather of fixed-size exported columns across the ranks of a
        node (include/madrona_b200.h, peer_gather.cu).  slots / shapes / dtypes describe
        this rank's columns; returns a PeerGather whose handle must be exchanged."""
        return PeerGather(self, slots, shapes, dtypes, world_size, rank)

    def snapshot(self) -> "Snapshot":
        """A device-memory snapshot of this executor's simulation state, empty until its
        first save() (include/madrona_b200.h)."""
        return Snapshot(self)

    def close(self) -> None:
        if self._h:
            # snapshots go before their executor
            for snap in list(getattr(self, "_snapshots", ())):
                snap.close()
            self._lib.mb2_executor_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Snapshot:
    """Every byte of an executor's device state that a later step can read, held in device
    memory: save() copies the live state in, restore() copies it back, each one kernel launch
    on `stream` (None: the executor's stream; a torch.cuda.Stream or a raw handle as runAsync
    takes it) without synchronizing the host.  Stepping after restore() reproduces what
    stepping after save() did, bit for bit.  Only the executor that made the snapshot can
    restore it; exported tensors keep their addresses and see the restored rows."""

    def __init__(self, ex: "MWCudaExecutor"):
        self._lib = ex._lib
        self._ex = ex
        self._h = None
        h = self._lib.mb2_snapshot_create(ex._h)
        if not h:
            raise MadronaB200Error(_last_error(self._lib))
        self._h = h
        ex._snapshots.add(self)

    def _call(self, name, stream):
        if not self._h:
            raise MadronaB200Error(f"snapshot {name}: the snapshot is closed")
        s = self._ex.stream if stream is None else int(getattr(stream, "cuda_stream", stream))
        if getattr(self._lib, f"mb2_snapshot_{name}")(self._ex._h, self._h, ctypes.c_void_p(s)) != 0:
            raise MadronaB200Error(_last_error(self._lib))

    def save(self, stream=None) -> None:
        self._call("save", stream)

    def restore(self, stream=None) -> None:
        self._call("restore", stream)

    @property
    def nbytes(self) -> int:
        """Bytes of device memory the snapshot holds (it grows when a save follows table growth)."""
        return int(self._lib.mb2_snapshot_bytes(self._h)) if self._h else 0

    @property
    def saved_nbytes(self) -> int:
        """Bytes the last save() copied: the live part of the state (waits for the device)."""
        return int(self._lib.mb2_snapshot_saved_bytes(self._h)) if self._h else 0

    def close(self) -> None:
        if self._h:
            if self._ex._h:
                self._lib.mb2_snapshot_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MeshBVHData:
    """BLAS of a set of triangle meshes in the reference's MeshBVHData format (role of
    render::AssetProcessor::makeBVHData): `view(device=True)` is what goes into
    CudaBatchRenderConfig.geoBVHData.  meshes: list of (positions [nv,3] f32, indices
    [nt,3] u32, material_idx) or (positions, indices, material_idx, uvs [nv,2] f32); meshes
    without uvs get (0, 0) at every vertex."""

    def __init__(self, meshes, gpu_id: int = -1):
        import numpy as np
        self._lib = load_library()
        self._keep = []
        srcs = (_MeshSourceC * len(meshes))()
        for i, mesh in enumerate(meshes):
            pos, idx, mat = mesh[:3]
            pos = np.ascontiguousarray(pos, dtype=np.float32)
            idx = np.ascontiguousarray(idx, dtype=np.uint32)
            uvs = None
            if len(mesh) > 3 and mesh[3] is not None:
                uvs = np.ascontiguousarray(mesh[3], dtype=np.float32)
                if uvs.shape != (len(pos), 2):
                    raise MadronaB200Error(f"mesh {i}: uvs must be [{len(pos)}, 2], got {list(uvs.shape)}")
            self._keep += [pos, idx, uvs]
            srcs[i] = _MeshSourceC(pos.ctypes.data, None if uvs is None else uvs.ctypes.data, len(pos),
                                   idx.ctypes.data, len(idx), int(mat))
        self.num_triangles = [len(m[1]) for m in meshes]
        self._h = self._lib.mb2_build_mesh_bvhs(srcs, len(meshes), gpu_id)
        if not self._h:
            raise MadronaB200Error(_last_error(self._lib))

    def view(self, device: bool = True) -> _MeshBVHViewC:
        return self._lib.mb2_mesh_bvh_data_view(self._h, 1 if device else 0).contents

    def triangle_sources(self):
        """For every triangle of the concatenated BLAS order: its index in its source mesh."""
        import numpy as np
        n = sum(self.num_triangles)
        ptr = self._lib.mb2_mesh_bvh_triangle_sources(self._h)
        return np.ctypeslib.as_array(ptr, shape=(n,)).copy()

    def host_arrays(self):
        """(nodes bytes [n,60], vertices f32 [nv,5], per-mesh (first_node, num_nodes, first_tri, num_tris, root box))."""
        import numpy as np
        v = self.view(device=False)
        nodes = np.ctypeslib.as_array(ctypes.cast(v.nodes, ctypes.POINTER(ctypes.c_uint8)),
                                      shape=(v.num_nodes, 60)).copy()
        verts = np.ctypeslib.as_array(ctypes.cast(v.vertices, ctypes.POINTER(ctypes.c_float)),
                                      shape=(v.num_verts, 5)).copy()
        return nodes, verts

    def close(self):
        if self._h:
            self._lib.mb2_mesh_bvh_data_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MaterialData:
    """Materials and textures in the reference's MaterialData format (role of
    render::AssetProcessor::initMaterialData): `view()` is what goes into
    CudaBatchRenderConfig.materialData.

    materials: list of (color rgba, texture_idx, roughness, metalness); texture_idx -1 = none.
    textures:  list of (data, format, width, height) == imp::SourceTexture, data a bytes-like
               buffer (RGBA8 rows, or BC7 16-byte blocks in rows of width / 4) or None.
    Executors adopt the pointers without owning them: close this after every executor
    that was created from it."""

    R8G8B8A8 = 0
    BC7 = 1

    def __init__(self, materials, textures=(), gpu_id: int = 0):
        import numpy as np
        self._lib = load_library()
        self._h = None
        self._keep = []
        c_tex = (_SourceTextureC * max(len(textures), 1))()
        for i, (data, fmt, width, height) in enumerate(textures):
            ptr, nbytes = None, 0
            if data is not None:
                buf = np.ascontiguousarray(np.frombuffer(memoryview(data).cast("B"), dtype=np.uint8))
                self._keep.append(buf)
                ptr, nbytes = buf.ctypes.data, buf.nbytes
            c_tex[i] = _SourceTextureC(ptr, int(fmt), int(width), int(height), nbytes)
        c_mat = (_SourceMaterialC * max(len(materials), 1))()
        for i, (color, tex_idx, roughness, metalness) in enumerate(materials):
            c_mat[i] = _SourceMaterialC((ctypes.c_float * 4)(*[float(c) for c in color]), int(tex_idx),
                                        float(roughness), float(metalness))
        self.num_textures = len(textures)
        self._h = self._lib.mb2_init_material_data(c_mat, len(materials), c_tex, len(textures), int(gpu_id))
        self._keep = None        # the pixels were copied to the device
        if not self._h:
            raise MadronaB200Error(_last_error(self._lib))

    def view(self) -> _MaterialViewC:
        return self._lib.mb2_material_data_view(self._h).contents

    def close(self):
        if self._h:
            self._lib.mb2_material_data_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RigidBodyAssets:
    """Physics asset pipeline (role of RigidBodyAssets::processRigidBodyAssets +
    PhysicsLoader::loadRigidBodies, include/madrona/physics_assets.hpp:30-66): convex hull
    meshes and collision objects in, a phys::ObjectManager out.

    hulls:   list of (positions [nv,3] f32, faces) -- faces a list of CCW vertex loops
    objects: list of dicts {"prims": [("sphere", r) | ("hull", idx) | ("plane",)],
                            "inv_mass": float, "mu_s": float, "mu_d": float}
    `device_ptr` is what a simulator's Config.rigidBodyObjectManager takes (gpu_id >= 0)."""

    TYPES = {"sphere": 1, "hull": 2, "plane": 4}

    def __init__(self, hulls, objects, gpu_id: int = -1):
        import numpy as np
        self._lib = load_library()
        keep = []
        c_hulls = (_SourceHullC * max(len(hulls), 1))()
        for i, (pos, faces) in enumerate(hulls):
            pos = np.ascontiguousarray(pos, dtype=np.float32)
            counts = np.asarray([len(f) for f in faces], dtype=np.uint32)
            idx = np.asarray([v for f in faces for v in f], dtype=np.uint32)
            keep += [pos, counts, idx]
            c_hulls[i] = _SourceHullC(pos.ctypes.data, len(pos), idx.ctypes.data, counts.ctypes.data, len(faces))
        c_objs = (_SourceObjectC * max(len(objects), 1))()
        for i, obj in enumerate(objects):
            prims = (_SourcePrimC * len(obj["prims"]))()
            for j, p in enumerate(obj["prims"]):
                prims[j] = _SourcePrimC(self.TYPES[p[0]], float(p[1]) if p[0] == "sphere" else 0.0,
                                        int(p[1]) if p[0] == "hull" else 0)
            keep.append(prims)
            c_objs[i] = _SourceObjectC(prims, len(obj["prims"]), float(obj["inv_mass"]),
                                       float(obj.get("mu_s", 0.5)), float(obj.get("mu_d", 0.5)))
        self._h = self._lib.mb2_process_rigid_body_assets(c_hulls, len(hulls), c_objs, len(objects), gpu_id)
        if not self._h:
            raise MadronaB200Error(_last_error(self._lib))
        self.gpu_id = gpu_id

    @property
    def device_ptr(self) -> int:
        p = self._lib.mb2_object_manager_ptr(self._h, 1)
        if not p:
            raise MadronaB200Error("RigidBodyAssets was built without a GPU (gpu_id < 0)")
        return int(p)

    def host_arrays(self) -> dict:
        """Copies of the host arrays, pointers in the primitives replaced by element offsets
        into the concatenated hull arrays."""
        import numpy as np
        v = _RigidBodyAssetsC()
        self._lib.mb2_object_manager_host_assets(self._h, ctypes.byref(v))

        def arr(ptr, n, width):
            if n == 0:
                return np.zeros((0, width), dtype=np.uint8)
            return np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_uint8)), shape=(n, width)).copy()
        prims_raw = arr(v.primitives, v.total_num_primitives, 56)
        prims = []
        for row in prims_raw:
            type_ = int(row[0:4].view(np.uint32)[0])
            if type_ == 1:
                prims.append((type_, float(row[8:12].view(np.float32)[0])))
            elif type_ == 2:
                ptrs = row[8:40].view(np.uint64)
                n = row[40:52].view(np.uint32)
                prims.append((type_, (int(ptrs[0]) - v.half_edges) // 12, (int(ptrs[1]) - v.face_base_half_edges) // 4,
                              (int(ptrs[3]) - v.vertices) // 12, int(n[0]), int(n[1]), int(n[2]),
                              (int(ptrs[2]) - v.face_planes) // 16))
            else:
                prims.append((type_,))
        return {
            "half_edges": arr(v.half_edges, v.num_half_edges, 12).view(np.uint32),
            "face_base": arr(v.face_base_half_edges, v.num_faces, 4).view(np.uint32).reshape(-1),
            "planes": arr(v.face_planes, v.num_faces, 16).view(np.float32),
            "vertices": arr(v.vertices, v.num_verts, 12).view(np.float32),
            "prims": prims,
            "prim_aabbs": arr(v.primitive_aabbs, v.total_num_primitives, 24).view(np.float32),
            "metadatas": arr(v.metadatas, v.num_objs, 52).view(np.float32),
            "obj_aabbs": arr(v.obj_aabbs, v.num_objs, 24).view(np.float32),
            "prim_offsets": arr(v.prim_offsets, v.num_objs, 4).view(np.uint32).reshape(-1),
            "prim_counts": arr(v.prim_counts, v.num_objs, 4).view(np.uint32).reshape(-1),
        }

    def close(self):
        if self._h:
            self._lib.mb2_object_manager_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Navmesh:
    """Host navmesh builder (the reference's host Navmesh::initFromPolygons, include/madrona/
    navmesh.hpp) for a mesh that many worlds share: the four arrays of a madrona::Navmesh,
    bit-identical to the reference's, built once and uploaded once to `gpu_id`
    (gpu_id < 0: host arrays only).

    vertices: [nv, 3] float32; polygons: a list of vertex-index loops (CCW, at least 3
    each; fanned from the first index) or a pair (flat indices, sizes) with the offsets
    implied, or a triple (flat indices, offsets, sizes).
    `view_bytes()` is the 40-byte madrona::Navmesh holding device pointers, to copy into a
    simulator's Config.  Executors adopt those pointers without owning them: close() the
    navmesh only after every executor that uses it."""

    def __init__(self, vertices, polygons, gpu_id: int = -1):
        import numpy as np
        self._lib = load_library()
        self._h = None
        verts = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
        if isinstance(polygons, tuple) and len(polygons) == 3:
            idx, offsets, sizes = (np.ascontiguousarray(a, dtype=np.uint32) for a in polygons)
        elif isinstance(polygons, tuple) and len(polygons) == 2:
            idx, sizes = (np.ascontiguousarray(a, dtype=np.uint32) for a in polygons)
            offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.uint32) if len(sizes) else sizes
        else:
            sizes = np.asarray([len(p) for p in polygons], dtype=np.uint32)
            idx = np.asarray([v for p in polygons for v in p], dtype=np.uint32)
            offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.uint32) if len(sizes) else sizes
        if len(offsets) != len(sizes):
            raise MadronaB200Error("Navmesh: offsets and sizes differ in length")
        # keep empty inputs non-null: the builder rejects them with its own message
        keep = [a if len(a) else np.zeros(1, dtype=a.dtype) for a in (verts.reshape(-1), idx, offsets, sizes)]
        self._h = self._lib.mb2_navmesh_create(keep[0].ctypes.data, len(verts), keep[1].ctypes.data, len(idx),
                                               keep[2].ctypes.data, keep[3].ctypes.data, len(sizes), int(gpu_id))
        if not self._h:
            raise MadronaB200Error(_last_error(self._lib))
        self.gpu_id = int(gpu_id)

    def view_bytes(self) -> bytes:
        """The 40-byte madrona::Navmesh (device pointers, numVerts, numTris)."""
        p = self._lib.mb2_navmesh_view(self._h)
        if not p:
            raise MadronaB200Error("Navmesh was built without a GPU (gpu_id < 0)")
        return ctypes.string_at(p, 40)

    def arrays(self) -> dict:
        """Copies of the host arrays: vertices [nv,3] f32, tri_indices and tri_adjacency
        [T,3] u32, alias_tau [T] f32 and alias [T] u32."""
        import numpy as np
        v = _NavmeshArraysC()
        self._lib.mb2_navmesh_host_arrays(self._h, ctypes.byref(v))

        def arr(ptr, n, dtype):
            if n == 0:
                return np.zeros(0, dtype=dtype)
            raw = ctypes.string_at(ptr, n * np.dtype(dtype).itemsize)
            return np.frombuffer(raw, dtype=dtype).copy()
        alias = arr(v.alias_table, 2 * v.num_tris, np.uint32).reshape(-1, 2)
        return {
            "vertices": arr(v.vertices, 3 * v.num_verts, np.float32).reshape(-1, 3),
            "tri_indices": arr(v.tri_indices, 3 * v.num_tris, np.uint32).reshape(-1, 3),
            "tri_adjacency": arr(v.tri_adjacency, 3 * v.num_tris, np.uint32).reshape(-1, 3),
            "alias_tau": alias[:, 0].copy().view(np.float32),
            "alias": alias[:, 1].copy(),
        }

    def close(self):
        if self._h:
            self._lib.mb2_navmesh_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PeerGather:
    """Symmetric-buffer gather: every rank pushes its exported columns into every
    peer's buffer with NVLink peer stores (one kernel per step), consumers wait on
    per-rank step flags.  See include/madrona_b200.h for the protocol."""

    HANDLE_BYTES = 128

    def __init__(self, ex: "MWCudaExecutor", slots, shapes, dtypes, world_size: int, rank: int):
        import numpy as np
        self._lib = ex._lib
        self._ex = ex
        self.world_size, self.rank = int(world_size), int(rank)
        self.shapes = [tuple(int(d) for d in s) for s in shapes]
        self.dtypes = list(dtypes)
        nbytes = [int(np.prod(s)) * np.dtype(d).itemsize for s, d in zip(self.shapes, self.dtypes)]
        c_slots = (ctypes.c_int64 * len(slots))(*[int(s) for s in slots])
        c_bytes = (ctypes.c_uint64 * len(slots))(*nbytes)
        self._h = self._lib.mb2_peer_gather_create(ex._h, c_slots, len(slots), c_bytes, self.world_size, self.rank)
        if not self._h:
            raise MadronaB200Error(_last_error(self._lib))

    def local_handle(self) -> bytes:
        buf = ctypes.create_string_buffer(self.HANDLE_BYTES)
        if self._lib.mb2_peer_gather_local_handle(self._h, buf) != 0:
            raise MadronaB200Error(_last_error(self._lib))
        return buf.raw

    def connect(self, all_handles: Sequence[bytes]) -> None:
        blob = b"".join(all_handles)
        assert len(blob) == self.HANDLE_BYTES * self.world_size
        if self._lib.mb2_peer_gather_connect(self._h, blob) != 0:
            raise MadronaB200Error(_last_error(self._lib))

    def _call(self, name, stream):
        s = getattr(stream, "cuda_stream", stream)
        if getattr(self._lib, f"mb2_peer_gather_{name}_async")(self._h, ctypes.c_void_p(int(s))) != 0:
            raise MadronaB200Error(f"peer gather {name} launch failed")

    def push(self, stream):
        self._call("push", stream)

    def wait(self, stream):
        self._call("wait", stream)

    def release(self, stream):
        self._call("release", stream)

    def tensor(self, parity: int, index: int):
        """World-major gathered column [world_size * W_local, ...] of a parity (zero copy)."""
        import torch
        shape = (self.world_size * self.shapes[index][0],) + self.shapes[index][1:]
        ptr = self._lib.mb2_peer_gather_buffer(self._h, int(parity), int(index))
        view = _CudaView(ptr, shape, _TYPESTR[self.dtypes[index]])
        return torch.as_tensor(view, device=f"cuda:{self._ex.gpu_id}")

    def close(self):
        if self._h:
            self._lib.mb2_peer_gather_destroy(self._h)
            self._h = None
