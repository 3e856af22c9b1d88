/* madrona_b200.h -- C ABI of libmadrona_b200.so, the H100-native drop-in for
 * the Madrona GPU backend (madrona::MWCudaExecutor).
 *
 * Every entry point cites the reference interface it replaces
 * (/root/reference = shacklettbp/madrona @ b31034bd).  Only plain C types
 * cross this boundary: no torch, no C++ classes.  The C++ facade with the
 * reference's exact class names (madrona::MWCudaExecutor, MWCudaLaunchGraph,
 * StateConfig, CompileConfig) is the header-only wrapper in
 * madrona_b200/host/madrona/mw_gpu.hpp; Python binds the same symbols with
 * ctypes (madrona_b200/executor.py).
 *
 * Error convention: the reference FATAL()s (print + abort,
 * include/madrona/crash.hpp).  The C ABI instead returns NULL / non-zero and
 * keeps a message retrievable with mb2_last_error(); the C++ facade turns
 * that back into print + abort so C++ callers see reference behaviour.
 */
#ifndef MADRONA_B200_H
#define MADRONA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mb2_executor mb2_executor;
typedef struct mb2_launch_graph mb2_launch_graph;

/* == madrona::StateConfig, include/madrona/mw_gpu.hpp:25-51 (same fields,
 * same order, same meaning; host pointers are copied during create). */
typedef struct mb2_state_config {
    const void *world_init_ptr;
    uint32_t num_world_init_bytes;
    const void *user_config_ptr;
    uint32_t num_user_config_bytes;
    uint32_t num_world_data_bytes;
    uint32_t world_data_alignment;
    uint32_t num_worlds;
    uint32_t num_taskgraphs;
    uint32_t num_exported_buffers;
} mb2_state_config;

/* == madrona::CompileConfig, include/madrona/mw_gpu.hpp:53-73.  user_sources
 * are the simulator's C++ files (the same files the reference NVRTC-compiles);
 * opt_mode: 0 Optimize, 1 LTO (treated as Optimize: single-module build),
 * 2 Debug. */
typedef struct mb2_compile_config {
    const char *const *user_sources;
    uint32_t num_user_sources;
    const char *const *user_compile_flags;
    uint32_t num_user_compile_flags;
    uint32_t opt_mode;
} mb2_compile_config;

/* == render::MeshBVHData / render::MaterialData
 * (include/madrona/render/cuda_batch_render_assets.hpp): DEVICE pointers to
 * reference-format arrays -- QBVHNode (60 B), MeshBVH::LeafMaterial,
 * MeshBVH::BVHVertex (20 B), MeshBVH (72 B), Material (28 B); layouts in
 * madrona_b200/csrc/render_bvh.h.  What render::AssetProcessor::makeBVHData
 * returns can be passed as is; mb2_build_mesh_bvhs builds the same from
 * triangle meshes. */
typedef struct mb2_mesh_bvh_view {
    void *nodes;
    uint64_t num_nodes;
    void *leaf_material;
    uint64_t num_leaves;
    void *vertices;
    uint64_t num_verts;
    void *mesh_bvhs;
    uint64_t num_bvhs;
} mb2_mesh_bvh_view;

typedef struct mb2_material_view {
    void *textures;                /* cudaTextureObject_t * (device): sampled by the RGBD ray caster */
    uint32_t num_texture_buffers;  /* entries of textures; a textureIdx at or above it fails the render */
    void *texture_buffers;         /* cudaArray_t * (host), owned by whoever built the textures */
    void *materials;               /* madrona::Material * (device) or NULL */
} mb2_material_view;

/* == madrona::CudaBatchRenderConfig, include/madrona/mw_gpu.hpp:75-96 (same
 * fields, same order), then the image size.  Each view's output is row-major
 * [render_height][render_width]: RGBA8 plus f32 depth (RGBD) or depth only.
 * Both 0 (what a caller that fills only the first six fields passes when it
 * zero-initialises the struct): a render_resolution square.  Set together; a
 * nonzero render_resolution must then equal both.  The vertical field of view
 * spans the rows, the horizontal one is widened by width / height.
 * render_width * render_height * 4 must fit in 32 bits.  mb2_executor_create
 * returns NULL and mb2_last_error() says why when any of this does not hold. */
typedef struct mb2_render_config {
    uint32_t render_mode;          /* 0 RGBD, 1 Depth */
    mb2_mesh_bvh_view geo_bvh_data;
    mb2_material_view material_data;
    uint32_t render_resolution;    /* square output, unless render_width / render_height are set */
    float near_plane;
    float far_plane;
    uint32_t render_width;         /* columns per view, or 0 */
    uint32_t render_height;        /* rows per view, or 0 */
} mb2_render_config;

/* Triangle mesh -> BLAS.  Role of MeshBVHBuilder (src/common/mesh_bvh_builder.cpp,
 * embree based) + render::AssetProcessor::makeBVHData (src/render/
 * asset_processor.cpp): one reference-format MeshBVH per mesh, arrays
 * concatenated, uploaded to gpu_id (gpu_id < 0: host only).  uvs may be NULL.
 * mb2_mesh_bvh_data_view returns a pointer to an mb2_mesh_bvh_view with device
 * (device != 0) or host pointers; mb2_mesh_bvh_triangle_sources maps every
 * triangle of the concatenated BLAS order back to its index in its source mesh. */
typedef struct mb2_mesh_source {
    const float *positions;        /* xyz per vertex */
    const float *uvs;              /* uv per vertex or NULL */
    uint32_t num_vertices;
    const uint32_t *indices;       /* 3 per triangle */
    uint32_t num_triangles;
    int32_t material_idx;          /* -1: none (white) */
} mb2_mesh_source;
typedef struct mb2_mesh_bvh_data mb2_mesh_bvh_data;
mb2_mesh_bvh_data *mb2_build_mesh_bvhs(const mb2_mesh_source *meshes, uint32_t num_meshes, int gpu_id);
const void *mb2_mesh_bvh_data_view(const mb2_mesh_bvh_data *data, int device);
const uint32_t *mb2_mesh_bvh_triangle_sources(const mb2_mesh_bvh_data *data);
void mb2_mesh_bvh_data_destroy(mb2_mesh_bvh_data *data);

/* Materials and textures -> render::MaterialData.  Role of
 * render::AssetProcessor::initMaterialData (src/render/asset_processor.cpp):
 * every texture becomes a cudaArray (uchar4, or BC7 blocks) behind a texture
 * object with the reference's descriptor -- wrap on both axes, linear
 * filtering, normalized float reads, normalized coordinates -- and the
 * materials are uploaded as madrona::Material.  Every input is checked before
 * the first CUDA call; on a bad one the call returns NULL and
 * mb2_last_error() says why.  mb2_material_data_view returns the
 * mb2_material_view that goes into mb2_render_config::material_data.  The
 * executor adopts those pointers without owning them: destroy the handle
 * (mb2_material_data_destroy: texture objects, arrays, device buffers) after
 * every executor that uses it. */
typedef struct mb2_source_texture {     /* == imp::SourceTexture */
    const void *data;                   /* RGBA8 rows, or BC7 blocks in rows of width / 4 */
    int32_t format;                     /* 0 R8G8B8A8, 1 BC7 (width, height multiples of 4) */
    uint32_t width;
    uint32_t height;
    uint64_t num_bytes;                 /* width * height * 4, or width * height (BC7) */
} mb2_source_texture;
typedef struct mb2_source_material {    /* == imp::SourceMaterial */
    float color[4];                     /* multiplies the texture's rgb */
    int32_t texture_idx;                /* -1: no texture */
    float roughness;
    float metalness;
} mb2_source_material;
typedef struct mb2_material_data mb2_material_data;
mb2_material_data *mb2_init_material_data(const mb2_source_material *materials, uint32_t num_materials,
                                          const mb2_source_texture *textures, uint32_t num_textures,
                                          int gpu_id);
const mb2_material_view *mb2_material_data_view(const mb2_material_data *data);
void mb2_material_data_destroy(mb2_material_data *data);

/* MWCudaExecutor::initCUDA(int gpu_id), mw_gpu.hpp:122 / cuda_exec.cpp:2315.
 * Returns 0 on success. */
int mb2_init_cuda(int gpu_id);

/* Same, also returning the device's primary CUcontext (what
 * MWCudaExecutor::initCUDA hands back to the Manager), and the inverse lookup
 * (context -> device ordinal; NULL -> the current device). */
int mb2_init_cuda_ctx(int gpu_id, void **cu_context_out);
int mb2_device_of_context(void *cu_context);

/* MWCudaExecutor::MWCudaExecutor(const StateConfig&, const CompileConfig&,
 * CUcontext, const Optional<CudaBatchRenderConfig>&), mw_gpu.hpp:125-129 /
 * cuda_exec.cpp:2333-2420.  render_cfg may be NULL. */
mb2_executor *mb2_executor_create(const mb2_state_config *state_cfg,
                                  const mb2_compile_config *compile_cfg,
                                  int gpu_id,
                                  const mb2_render_config *render_cfg);

/* ~MWCudaExecutor(), mw_gpu.hpp:132. */
void mb2_executor_destroy(mb2_executor *exec);

/* MWCudaExecutor::buildLaunchGraph(Span<const uint32_t>, const char*),
 * mw_gpu.hpp:144-145 / cuda_exec.cpp:2174-2291. */
mb2_launch_graph *mb2_build_launch_graph(mb2_executor *exec,
                                         const uint32_t *taskgraph_ids,
                                         uint32_t num_taskgraphs,
                                         const char *stat_name);

/* MWCudaExecutor::buildLaunchGraphAllTaskGraphs(), mw_gpu.hpp:147. */
mb2_launch_graph *mb2_build_launch_graph_all(mb2_executor *exec);

/* MWCudaExecutor::buildRenderGraph(), mw_gpu.hpp:150 / cuda_exec.cpp:2527. */
mb2_launch_graph *mb2_build_render_graph(mb2_executor *exec);

/* ~MWCudaLaunchGraph(), mw_gpu.hpp:104. */
void mb2_launch_graph_destroy(mb2_launch_graph *graph);

/* MWCudaExecutor::run(MWCudaLaunchGraph&), mw_gpu.hpp:153 /
 * cuda_exec.cpp:2756-2794: launch + synchronise.  Returns 0 on success. */
int mb2_run(mb2_executor *exec, mb2_launch_graph *graph);

/* MWCudaExecutor::runAsync(MWCudaLaunchGraph&, cudaStream_t), mw_gpu.hpp:155
 * / cuda_exec.cpp:2796-2800: enqueue only; cuda_stream is a cudaStream_t.
 * The launch graphs of ONE executor share its ECS tables and the sort scratch
 * (tickets, histograms, look-back flags): they must be ordered with respect to
 * each other -- launch them on one stream, or chain the streams with events.
 * Two graphs of the same executor in flight at once is undefined (the
 * reference's megakernel has the same single-launch-at-a-time rule). */
int mb2_run_async(mb2_executor *exec, mb2_launch_graph *graph,
                  void *cuda_stream);

/* MWCudaExecutor::getExported(CountT slot), mw_gpu.hpp:159: borrowed device
 * pointer, stable for the executor's lifetime. */
void *mb2_get_exported(const mb2_executor *exec, int64_t slot);

/* ---- additions with no reference counterpart (introspection) ------------ */

/* Message of the last failed call on this thread ("" if none). */
const char *mb2_last_error(void);

/* Live row count of the table behind an export slot (device sync + read). */
int64_t mb2_get_exported_num_rows(mb2_executor *exec, int64_t slot);

/* Bytes per row of the exported component. */
int64_t mb2_get_exported_row_bytes(const mb2_executor *exec, int64_t slot);

/* With MADRONA_B200_RENDER_DEBUG=1 at executor creation: device pointer to
 * int32 [views][res * res][2] = (instance index inside its world, triangle
 * index inside the instance's mesh BLAS order) of every pixel's closest hit,
 * -1 for a miss; NULL otherwise.  Test hook of the ray caster. */
void *mb2_render_debug_hits(mb2_executor *exec);

/* Test hook: the ray caster's per-world structures of the last render-prepare.
 * The layouts are compact: world w's instances and TLAS nodes start at entry
 * offsets[w] of one list (offsets = exclusive scan of the instance counts).
 * which = 1: QBVHNode list (world w's tree at offsets[w], node 0 = root), 2: int32
 * TLAS node counts [worlds], 3: instance list (76-byte records: position,
 * rotation, scale, matID, objectID, colour, world box), 4: int32 instance counts
 * [worlds], 5: int32 instance offsets [worlds].  *stride is set to 0 (there is
 * no per-world stride).  Device pointers; NULL without a renderer. */
void *mb2_render_debug_buffer(mb2_executor *exec, int which, int64_t *stride);

/* Kernel nodes inside a built launch graph (== launches per run). */
int64_t mb2_launch_graph_num_kernels(const mb2_launch_graph *graph);

/* Capture streams the launch graph was built from: > 1 means TaskGraph nodes
 * that do not depend on each other (TaskGraphBuilder::addToGraph dependency
 * lists, include/madrona/taskgraph_builder.hpp:128-140) became parallel
 * branches of the CUDA graph. */
int64_t mb2_launch_graph_num_branches(const mb2_launch_graph *graph);

/* The stream mb2_run launches on (cudaStream_t). */
void *mb2_executor_stream(mb2_executor *exec);

/* Compile the simulator module for sm_90a without touching a GPU and store
 * it in the kernel cache (used by the build step on a CPU-only box).
 * Returns 0 on success. */
int mb2_jit_precompile(const mb2_compile_config *compile_cfg);

/* Per-node device timing (CUDA events on the executor's stream) of the task
 * graphs in taskgraph_ids, averaged over `reps` steps; this ADVANCES the
 * simulation by `reps` steps.  Replaces the reference's device tracing
 * (src/mw/device/include/madrona/mw_gpu/tracing.hpp, scripts/
 * parse_device_tracing.py).  Writes a JSON array of
 * {"node","kind","archetype","launches","ms","rows","bytes"} into json_out
 * ("bytes" = algorithmic bytes per launch, SURVEY.md 8d).  Returns the number
 * of characters needed (excluding NUL), or -1 on error. */
int64_t mb2_profile_nodes(mb2_executor *exec, const uint32_t *taskgraph_ids,
                          uint32_t num_taskgraphs, uint32_t reps,
                          char *json_out, uint64_t json_capacity);

/* ---- physics assets (SURVEY.md 8f N2) --------------------------------------
 * Role of RigidBodyAssets::processRigidBodyAssets (include/madrona/
 * physics_assets.hpp:11-66, src/physics/physics_assets.cpp:1268-1407, with
 * build_convex_hulls = false) + PhysicsLoader::loadRigidBodies /
 * getObjectManager (include/madrona/physics_loader.hpp): convex hull meshes
 * (polygon faces, coplanar faces merged) and collision objects in, the
 * phys::ObjectManager a simulator's Config points at out -- half-edge meshes,
 * Newell face planes, primitive / object AABBs, mass properties with the
 * inertia tensor diagonalised -- on the host and, for gpu_id >= 0, on the GPU.
 * Primitive types: 1 sphere, 2 hull, 4 plane (CollisionPrimitive::Type). */
typedef struct mb2_source_hull {        /* == imp::SourceMesh as physics uses it */
    const float *positions;             /* xyz per vertex */
    uint32_t num_vertices;
    const uint32_t *indices;            /* concatenated face loops */
    const uint32_t *face_counts;        /* vertices per face; NULL: triangles */
    uint32_t num_faces;
} mb2_source_hull;
typedef struct mb2_source_prim {        /* == phys::SourceCollisionPrimitive */
    uint32_t type;
    float sphere_radius;
    uint32_t hull_idx;
} mb2_source_prim;
typedef struct mb2_source_object {      /* == phys::SourceCollisionObject */
    const mb2_source_prim *prims;
    uint32_t num_prims;
    float inv_mass;
    float mu_s, mu_d;
} mb2_source_object;
typedef struct mb2_object_manager mb2_object_manager;
mb2_object_manager *mb2_process_rigid_body_assets(const mb2_source_hull *hulls, uint32_t num_hulls,
                                                  const mb2_source_object *objects, uint32_t num_objects,
                                                  int gpu_id);
/* phys::ObjectManager * valid on the device (device != 0: what goes into the
 * simulator's Config) or on the host */
void *mb2_object_manager_ptr(const mb2_object_manager *mgr, int device);
/* == phys::RigidBodyAssets (physics_assets.hpp:30-56): the host arrays behind the
 * manager (hull arrays concatenated over hulls; primitives hold host pointers) */
typedef struct mb2_rigid_body_assets {
    void *half_edges;               /* geo::HalfEdge {next, rootVertex, face} */
    uint32_t *face_base_half_edges;
    void *face_planes;              /* geo::Plane {normal, d} */
    void *vertices;                 /* math::Vector3 */
    uint32_t num_half_edges, num_faces, num_verts;
    void *primitives;               /* phys::CollisionPrimitive (56 B) */
    void *primitive_aabbs;          /* math::AABB */
    void *metadatas;                /* phys::RigidBodyMetadata (52 B) */
    void *obj_aabbs;
    uint32_t *prim_offsets;
    uint32_t *prim_counts;
    uint32_t num_convex_hulls, total_num_primitives, num_objs;
} mb2_rigid_body_assets;
void mb2_object_manager_host_assets(const mb2_object_manager *mgr, mb2_rigid_body_assets *out);
void mb2_object_manager_destroy(mb2_object_manager *mgr);

/* ---- navigation meshes -----------------------------------------------------
 * Role of the reference's host Navmesh::initFromPolygons (include/madrona/
 * navmesh.hpp, src/common/navmesh.cpp) for a mesh that many worlds share:
 * polygons (CCW vertex loops, fanned from their first index) in, the four
 * arrays of a madrona::Navmesh out, bit-identical to the reference's, uploaded
 * once to gpu_id (gpu_id < 0: host arrays only).  Bad input returns NULL and
 * mb2_last_error() says why: a null array, no polygons, a polygon of fewer
 * than 3 vertices, one running past num_idxs, or an index >= num_verts.
 * mb2_navmesh_view returns a host copy of the 40-byte madrona::Navmesh that
 * holds the device pointers, to copy into a simulator's Config (NULL without a
 * GPU).  Executors adopt those pointers without owning them: destroy the
 * navmesh after every executor that uses it. */
typedef struct mb2_navmesh mb2_navmesh;
typedef struct mb2_navmesh_arrays {
    const float *vertices;              /* xyz per vertex */
    const uint32_t *tri_indices;        /* 3 per triangle */
    const uint32_t *tri_adjacency;      /* 3 per triangle, edge (a,b) (b,c) (c,a); 0xFFFFFFFF: none */
    const void *alias_table;            /* Navmesh::AliasEntry {float tau; uint32_t alias} per triangle */
    uint32_t num_verts;
    uint32_t num_tris;
} mb2_navmesh_arrays;
mb2_navmesh *mb2_navmesh_create(const float *vertices_xyz, uint32_t num_verts,
                                const uint32_t *poly_idxs, uint32_t num_idxs,
                                const uint32_t *poly_offsets, const uint32_t *poly_sizes,
                                uint32_t num_polys, int gpu_id);
const void *mb2_navmesh_view(const mb2_navmesh *navmesh);
void mb2_navmesh_host_arrays(const mb2_navmesh *navmesh, mb2_navmesh_arrays *out);
void mb2_navmesh_destroy(mb2_navmesh *navmesh);

/* ---- multi-GPU gather of exported columns (SURVEY.md 8e) ------------------
 * No reference counterpart (the reference is single-GPU, mw_gpu.hpp:122):
 * worlds shard across GPUs, one process per GPU, and the only exchange is the
 * gather of exported tensors (observations, rewards, dones) into the
 * world-major tensor every rank sees.  Instead of one NCCL all_gather per
 * tensor per step, each rank pushes its slices straight into every peer's
 * symmetric buffer with NVLink peer stores from one kernel (peer_gather.cu).
 *
 *   g = mb2_peer_gather_create(exec, slots, n, bytes_per_slot, world_size, rank)
 *   mb2_peer_gather_local_handle(g, h)      -> 128 opaque bytes; exchange them
 *   mb2_peer_gather_connect(g, all)         <- world_size * 128 bytes, rank order
 *   per step:  run_async(graph); push_async(g); ... wait_async(g); read
 *              mb2_peer_gather_buffer(g, step & 1, i); release_async(g)
 * push / wait / release each advance their own step counter (kept on the
 * device), so they are CUDA-graph friendly.  bytes_per_slot[i] = bytes of ONE
 * rank's column (identical on all ranks, multiple of 4); buffer i of a parity
 * is [world_size][bytes_per_slot[i]], i.e. the world-major gathered column. */
typedef struct mb2_peer_gather mb2_peer_gather;
#define MB2_PEER_GATHER_HANDLE_BYTES 128
mb2_peer_gather *mb2_peer_gather_create(mb2_executor *exec, const int64_t *slots,
                                        uint32_t num_slots, const uint64_t *bytes_per_slot,
                                        uint32_t world_size, uint32_t rank);
int mb2_peer_gather_local_handle(mb2_peer_gather *gather, void *handle_out);
int mb2_peer_gather_connect(mb2_peer_gather *gather, const void *all_handles);
int mb2_peer_gather_push_async(mb2_peer_gather *gather, void *cuda_stream);
int mb2_peer_gather_wait_async(mb2_peer_gather *gather, void *cuda_stream);
int mb2_peer_gather_release_async(mb2_peer_gather *gather, void *cuda_stream);
void *mb2_peer_gather_buffer(mb2_peer_gather *gather, uint32_t parity, uint32_t slot_index);
void mb2_peer_gather_destroy(mb2_peer_gather *gather);

/* ---- snapshots of an executor's simulation state ----------------------------
 * No reference counterpart.  A snapshot is a device buffer that holds every
 * byte of device state a later launch graph can read: the live rows of every
 * table, the entity store, world data, the persistent and tmp arenas, custom
 * node data and the ray caster's last prepared scene.  save copies the live
 * state into it, restore copies it back; each is one kernel launch on
 * cuda_stream (NULL: the legacy default stream), ordered like run_async and
 * never synchronizing the host.  Stepping after a restore reproduces, bit for
 * bit, what stepping after the save did.
 *   - a snapshot belongs to the executor that created it: save / restore with
 *     another executor, restore before any save, and null handles fail with a
 *     message in mb2_last_error() (return 1) and launch nothing;
 *   - it is sized for the table capacities at creation; a save after a table
 *     grew enlarges it first (stream-ordered), a restore always fits;
 *   - it shares the executor's tables, so it is part of the "one launch graph
 *     in flight" rule: order saves and restores with the executor's launches;
 *   - destroy snapshots before their executor; destroy waits for the device.
 * mb2_snapshot_bytes is the size of the buffer, which holds every table and
 * arena at its capacity; mb2_snapshot_saved_bytes is what the last save
 * copied, the live part (0 before a save; it waits for the device).  Both
 * return -1 for a null handle. */
typedef struct mb2_snapshot mb2_snapshot;
mb2_snapshot *mb2_snapshot_create(mb2_executor *exec);
int mb2_snapshot_save(mb2_executor *exec, mb2_snapshot *snap, void *cuda_stream);
int mb2_snapshot_restore(mb2_executor *exec, mb2_snapshot *snap, void *cuda_stream);
int64_t mb2_snapshot_bytes(const mb2_snapshot *snap);
int64_t mb2_snapshot_saved_bytes(mb2_snapshot *snap);
void mb2_snapshot_destroy(mb2_snapshot *snap);

/* Version string. */
const char *mb2_version(void);

#ifdef __cplusplus
}
#endif

#endif
