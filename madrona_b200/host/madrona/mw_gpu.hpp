// madrona::MWCudaExecutor -- host-side C++ facade with the reference's class
// names, constructor and method signatures (include/madrona/mw_gpu.hpp:25-164),
// implemented as a thin header-only wrapper over the C ABI of
// libmadrona_b200.so (include/madrona_b200.h).  A simulator's Manager
// (mgr.cpp) that was written against the reference compiles against this
// header unchanged and links with -lmadrona_b200 instead of madrona_mw_gpu.
//
// Error convention: like the reference, failures print a message and abort
// (reference FATAL(), include/madrona/crash.hpp).
#pragma once

#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <type_traits>
#include <utility>

#include "../../../include/madrona_b200.h"

typedef struct CUctx_st *CUcontext;
typedef struct CUstream_st *cudaStream_t;

// A Manager usually includes other reference headers too (utils, span, optional,
// importer, render assets).  When the reference's include directory is on the
// include path (after this one), its own definitions are used; only what is
// missing is declared here, with the reference's names and layouts.
#if __has_include(<madrona/span.hpp>)
#include <madrona/types.hpp>
#include <madrona/span.hpp>
#include <madrona/optional.hpp>
#define MB2_FACADE_HAS_REFERENCE_CORE 1
#endif
#if __has_include(<madrona/render/cuda_batch_render_assets.hpp>) && __has_include(<cuda_runtime.h>)
#include <madrona/render/cuda_batch_render_assets.hpp>
#define MB2_FACADE_HAS_REFERENCE_RENDER 1
#endif

namespace madrona {

#ifndef MB2_FACADE_HAS_REFERENCE_CORE
using CountT = int64_t;

template <typename T>
concept EnumType = std::is_enum_v<T>;

template <typename T>
class Span {
public:
    constexpr Span(T *ptr, CountT n) : ptr_(ptr), n_(n) {}
    template <CountT N>
    constexpr Span(T (&arr)[N]) : ptr_(arr), n_(N) {}
    constexpr T *data() const { return ptr_; }
    constexpr CountT size() const { return n_; }
    constexpr T &operator[](CountT i) const { return ptr_[i]; }
    constexpr T *begin() const { return ptr_; }
    constexpr T *end() const { return ptr_ + n_; }
private:
    T *ptr_;
    CountT n_;
};

template <typename T>
class Optional {
public:
    static Optional none() { return Optional(); }
    Optional() : has_(false) {}
    Optional(const T &v) : v_(v), has_(true) {}
    bool has_value() const { return has_; }
    const T &operator*() const { return v_; }
    const T *operator->() const { return &v_; }
private:
    T v_ {};
    bool has_;
};
#endif

#ifndef MB2_FACADE_HAS_REFERENCE_RENDER
// == include/madrona/render/cuda_batch_render_assets.hpp (pointers are device
// pointers to reference-format arrays, see madrona_b200/csrc/render_bvh.h)
namespace render {
struct MeshBVHData {
    void *nodes;
    uint64_t numNodes;
    void *leafMaterial;
    uint64_t numLeaves;
    void *vertices;
    uint64_t numVerts;
    void *meshBVHs;
    uint64_t numBVHs;
};
struct MaterialData {
    void *textures;
    uint32_t numTextureBuffers;
    void *textureBuffers;
    void *materials;
};
}
#endif

// == include/madrona/mw_gpu.hpp:25-51
struct StateConfig {
    void *worldInitPtr;
    uint32_t numWorldInitBytes;
    void *userConfigPtr;
    uint32_t numUserConfigBytes;
    uint32_t numWorldDataBytes;
    uint32_t worldDataAlignment;
    uint32_t numWorlds;
    uint32_t numTaskGraphs;
    uint32_t numExportedBuffers;
};

// == include/madrona/mw_gpu.hpp:53-73
struct CompileConfig {
    enum class OptMode : uint32_t {
        Optimize,
        LTO,
        Debug,
    };
    Span<const char * const> userSources;
    Span<const char * const> userCompileFlags;
    OptMode optMode = OptMode::LTO;
};

// == include/madrona/mw_gpu.hpp:75-96
struct CudaBatchRenderConfig {
    enum class RenderMode : uint32_t {
        RGBD,
        Depth,
    };
    RenderMode renderMode;
    render::MeshBVHData geoBVHData;
    render::MaterialData materialData;
    uint32_t renderResolution = 0;
    float nearPlane = 0.f;
    float farPlane = 0.f;
};

}

namespace madrona { class MWCudaExecutor; }

namespace madrona_b200 {
// Image size of every view for the MWCudaExecutor constructor overload that takes one:
// row-major [height][width] pixels, the vertical field of view spanning the rows.  Given
// with a CudaBatchRenderConfig whose renderResolution is 0 (or equal to both).
struct RenderImageSize {
    uint32_t width;
    uint32_t height;
};

// Outputs beyond RGB and depth for the MWCudaExecutor constructor overload that takes them.
// segmentation: every view also gets a row-major [height][width] int32 image, the Entity id
// (without its generation) of the renderable each pixel's primary ray hits first, -1 where
// it hits nothing.  Exported like the other outputs, through
// exportColumn<render::RaycastOutputArchetype, render::SegmentationOutputBuffer>.
// normals: every view also gets a row-major [height][width] image of int8 x, y, z, w, the
// unit geometric normal of the hit triangle times 127 in the view's frame (+x toward increasing
// column, +y toward increasing row, +z away from the camera), turned to face the camera, w = 0;
// all zero where the ray hits nothing.  Exported through
// exportColumn<render::RaycastOutputArchetype, render::NormalOutputBuffer>.
struct RenderOutputs {
    bool segmentation;
    bool normals;
};

// The camera model of every view, for the MWCudaExecutor constructor overload that takes one.
// Pinhole: the reference's camera.  Panorama: each view's image covers 360 degrees of azimuth
// across its columns (the middle looks along the view's forward, the seam is behind it) and
// the vertical field of view across its rows, evenly spaced in elevation; the depth output is
// the distance along the unit ray, a lidar's range.
enum class RenderProjection : uint32_t {
    Pinhole = 0,
    Panorama = 1,
};

// A view for MWCudaExecutor::renderFreeViews (== mb2_free_view): the world, the camera's world
// position (entity position plus camera offset), the viewing entity's Rotation (w, x, y, z; the
// camera looks along the rotated +y axis) and the vertical field of view, as attachEntityToView
// takes it.
struct FreeView {
    int32_t world;
    float position[3];
    float rotation[4];
    float vfovDegrees;
};

// Device pointers, or nullptr for an output not wanted, in the exported columns' layouts with
// view i at slice i: rgb uint8 [n][H][W][4], depth float [n][H][W], segmentation int32 [n][H][W],
// normals int8 [n][H][W][4].
struct FreeViewOutputs {
    void *rgb;
    void *depth;
    void *segmentation;
    void *normals;
};

// Rays for MWCudaExecutor::tracePhysicsRays (== mb2_physics_rays): device pointers, SoA and
// contiguous -- world int32 [n], origin float [n][3], direction float [n][3] (not normalised),
// max_t float [n] or nullptr for +inf.
struct PhysicsRays {
    const int32_t *world;
    const float *origin;
    const float *direction;
    const float *maxT;
};

// Device pointers, or nullptr for an output not wanted: entity int32 [n][2] {gen, id}
// (Entity::none() on a miss), t float [n] (0 on a miss), normal float [n][3] (world frame,
// 0 on a miss).
struct PhysicsRayHits {
    int32_t *entity;
    float *t;
    float *normal;
};

// A device-memory snapshot of an executor's simulation state (include/madrona_b200.h),
// made by MWCudaExecutor::snapshot().  save() / restore() are one kernel launch each on
// `strm` (by default the executor's stream) and never synchronize the host; stepping after
// restore() reproduces what stepping after save() did.  Destroy it before its executor.
class ExecutorSnapshot {
public:
    ExecutorSnapshot() : exec_(nullptr), h_(nullptr) {}
    ExecutorSnapshot(ExecutorSnapshot &&o) : exec_(o.exec_), h_(o.h_) { o.h_ = nullptr; }
    ~ExecutorSnapshot() { if (h_) mb2_snapshot_destroy(h_); }
    ExecutorSnapshot &operator=(ExecutorSnapshot &&o)
    {
        if (this != &o) {
            if (h_) mb2_snapshot_destroy(h_);
            exec_ = o.exec_;
            h_ = o.h_;
            o.h_ = nullptr;
        }
        return *this;
    }

    inline void save(cudaStream_t strm);
    inline void restore(cudaStream_t strm);
    void save() { save((cudaStream_t)mb2_executor_stream(exec_)); }
    void restore() { restore((cudaStream_t)mb2_executor_stream(exec_)); }
    // bytes of device memory the snapshot holds
    int64_t bytes() const { return mb2_snapshot_bytes(h_); }

private:
    ExecutorSnapshot(mb2_executor *exec, mb2_snapshot *h) : exec_(exec), h_(h) {}
    mb2_executor *exec_;
    mb2_snapshot *h_;
friend class ::madrona::MWCudaExecutor;
};
}

namespace madrona {

namespace detail {
[[noreturn]] inline void fatal(const char *what)
{
    fprintf(stderr, "madrona_b200: %s: %s\n", what, mb2_last_error());
    fflush(stderr);
    abort();
}
}

class MWCudaExecutor;

class MWCudaLaunchGraph {
public:
    MWCudaLaunchGraph() : h_(nullptr) {}
    MWCudaLaunchGraph(MWCudaLaunchGraph &&o) : h_(o.h_) { o.h_ = nullptr; }
    ~MWCudaLaunchGraph() { if (h_) mb2_launch_graph_destroy(h_); }
    MWCudaLaunchGraph &operator=(MWCudaLaunchGraph &&o)
    {
        if (this != &o) {
            if (h_) mb2_launch_graph_destroy(h_);
            h_ = o.h_;
            o.h_ = nullptr;
        }
        return *this;
    }
private:
    explicit MWCudaLaunchGraph(mb2_launch_graph *h) : h_(h) {}
    mb2_launch_graph *h_;
friend class MWCudaExecutor;
};

class MWCudaExecutor {
public:
    // Initializes CUDA, sets the current device and returns the device's primary
    // context (the reference creates its own context, cuda_exec.cpp:2315-2331;
    // this engine runs on the runtime's primary context so torch can share it).
    static CUcontext initCUDA(int gpu_id)
    {
        void *ctx = nullptr;
        if (mb2_init_cuda_ctx(gpu_id, &ctx) != 0) detail::fatal("initCUDA");
        return (CUcontext)ctx;
    }

    MWCudaExecutor() : h_(nullptr) {}

    MWCudaExecutor(const StateConfig &state_cfg, const CompileConfig &compile_cfg,
                   CUcontext cu_ctx,
                   const Optional<CudaBatchRenderConfig> &render_cfg =
                       Optional<CudaBatchRenderConfig>::none())
    {
        create(state_cfg, compile_cfg, cu_ctx, render_cfg, ::madrona_b200::RenderImageSize { 0, 0 },
               ::madrona_b200::RenderOutputs { false }, ::madrona_b200::RenderProjection::Pinhole);
    }

    // Not in the reference: the batch renderer's images are image_size.width columns by
    // image_size.height rows instead of renderResolution squared.
    MWCudaExecutor(const StateConfig &state_cfg, const CompileConfig &compile_cfg,
                   CUcontext cu_ctx, const Optional<CudaBatchRenderConfig> &render_cfg,
                   const ::madrona_b200::RenderImageSize &image_size)
    {
        create(state_cfg, compile_cfg, cu_ctx, render_cfg, image_size, ::madrona_b200::RenderOutputs { false },
               ::madrona_b200::RenderProjection::Pinhole);
    }

    // Not in the reference: the image size as above (RenderImageSize { 0, 0 }: the
    // renderResolution square) and the extra outputs every view gets.
    MWCudaExecutor(const StateConfig &state_cfg, const CompileConfig &compile_cfg,
                   CUcontext cu_ctx, const Optional<CudaBatchRenderConfig> &render_cfg,
                   const ::madrona_b200::RenderImageSize &image_size,
                   const ::madrona_b200::RenderOutputs &outputs)
    {
        create(state_cfg, compile_cfg, cu_ctx, render_cfg, image_size, outputs,
               ::madrona_b200::RenderProjection::Pinhole);
    }

    // Not in the reference: the image size and outputs as above, and the camera model of
    // every view (RenderProjection::Panorama: 360-degree equirectangular views).
    MWCudaExecutor(const StateConfig &state_cfg, const CompileConfig &compile_cfg,
                   CUcontext cu_ctx, const Optional<CudaBatchRenderConfig> &render_cfg,
                   const ::madrona_b200::RenderImageSize &image_size,
                   const ::madrona_b200::RenderOutputs &outputs,
                   ::madrona_b200::RenderProjection projection)
    {
        create(state_cfg, compile_cfg, cu_ctx, render_cfg, image_size, outputs, projection);
    }

    MWCudaExecutor(MWCudaExecutor &&o) : h_(o.h_) { o.h_ = nullptr; }
    ~MWCudaExecutor() { if (h_) mb2_executor_destroy(h_); }
    MWCudaExecutor &operator=(MWCudaExecutor &&o)
    {
        if (this != &o) {
            if (h_) mb2_executor_destroy(h_);
            h_ = o.h_;
            o.h_ = nullptr;
        }
        return *this;
    }

    template <EnumType EnumT>
    inline MWCudaLaunchGraph buildLaunchGraph(EnumT taskgraph_id, const char *stat_name = nullptr)
    {
        return buildLaunchGraph(static_cast<uint32_t>(taskgraph_id), stat_name);
    }

    inline MWCudaLaunchGraph buildLaunchGraph(uint32_t taskgraph_id, const char *stat_name = nullptr)
    {
        return buildLaunchGraph(Span<const uint32_t>(&taskgraph_id, 1), stat_name);
    }

    MWCudaLaunchGraph buildLaunchGraph(Span<const uint32_t> taskgraph_ids,
                                       const char *stat_name = nullptr)
    {
        mb2_launch_graph *g = mb2_build_launch_graph(h_, taskgraph_ids.data(),
                                                     (uint32_t)taskgraph_ids.size(), stat_name);
        if (!g) detail::fatal("buildLaunchGraph");
        return MWCudaLaunchGraph(g);
    }

    MWCudaLaunchGraph buildLaunchGraphAllTaskGraphs()
    {
        mb2_launch_graph *g = mb2_build_launch_graph_all(h_);
        if (!g) detail::fatal("buildLaunchGraphAllTaskGraphs");
        return MWCudaLaunchGraph(g);
    }

    MWCudaLaunchGraph buildRenderGraph()
    {
        mb2_launch_graph *g = mb2_build_render_graph(h_);
        if (!g) detail::fatal("buildRenderGraph");
        return MWCudaLaunchGraph(g);
    }

    void run(MWCudaLaunchGraph &launch_graph)
    {
        if (mb2_run(h_, launch_graph.h_) != 0) detail::fatal("run");
    }

    void runAsync(MWCudaLaunchGraph &launch_graph, cudaStream_t strm)
    {
        if (mb2_run_async(h_, launch_graph.h_, (void *)strm) != 0) detail::fatal("runAsync");
    }

    void *getExported(CountT slot) const { return mb2_get_exported(h_, (int64_t)slot); }

    // Not in the reference: ray-cast `views` of the scene the last step prepared into the
    // caller's buffers, every view image_size pixels with `projection`, enqueued on `strm`
    // (nullptr: the executor's stream) like runAsync (include/madrona_b200.h,
    // mb2_render_free_views).  A view with a camera's pose, field of view, size and projection
    // writes the render graph's bytes for that camera.
    void renderFreeViews(Span<const ::madrona_b200::FreeView> views, ::madrona_b200::RenderImageSize image_size,
                         ::madrona_b200::RenderProjection projection, ::madrona_b200::FreeViewOutputs outputs,
                         cudaStream_t strm = nullptr)
    {
        static_assert(sizeof(::madrona_b200::FreeView) == sizeof(mb2_free_view) &&
                      offsetof(::madrona_b200::FreeView, vfovDegrees) == offsetof(mb2_free_view, vfov_degrees),
                      "FreeView layout");
        const mb2_free_view_outputs out { outputs.rgb, outputs.depth, outputs.segmentation, outputs.normals };
        if (mb2_render_free_views(h_, (const mb2_free_view *)views.data(), (uint32_t)views.size(), image_size.width,
                                  image_size.height, (uint32_t)projection, &out, (void *)strm) != 0) {
            detail::fatal("renderFreeViews");
        }
    }

    // Not in the reference: trace n rays against the worlds' collision geometry as the last step
    // left it, enqueued on `strm` (nullptr: the executor's stream) like runAsync
    // (include/madrona_b200.h, mb2_trace_physics_rays).  Ray i gives what
    // BVH::traceRay(origin[i], direction[i], &t, &normal, max_t[i]) returns in world world[i].
    void tracePhysicsRays(::madrona_b200::PhysicsRays rays, uint32_t n, ::madrona_b200::PhysicsRayHits hits,
                          cudaStream_t strm = nullptr)
    {
        const mb2_physics_rays r { rays.world, rays.origin, rays.direction, rays.maxT };
        const mb2_physics_ray_hits h { hits.entity, hits.t, hits.normal };
        if (mb2_trace_physics_rays(h_, &r, n, &h, (void *)strm) != 0) detail::fatal("tracePhysicsRays");
    }

    // Not in the reference: a snapshot of this executor's state (empty until its first save)
    ::madrona_b200::ExecutorSnapshot snapshot()
    {
        mb2_snapshot *s = mb2_snapshot_create(h_);
        if (!s) detail::fatal("snapshot");
        return ::madrona_b200::ExecutorSnapshot(h_, s);
    }

private:
    void create(const StateConfig &state_cfg, const CompileConfig &compile_cfg, CUcontext cu_ctx,
                const Optional<CudaBatchRenderConfig> &render_cfg,
                const ::madrona_b200::RenderImageSize &image_size,
                const ::madrona_b200::RenderOutputs &outputs,
                ::madrona_b200::RenderProjection projection)
    {
        mb2_state_config sc {
            state_cfg.worldInitPtr, state_cfg.numWorldInitBytes,
            state_cfg.userConfigPtr, state_cfg.numUserConfigBytes,
            state_cfg.numWorldDataBytes, state_cfg.worldDataAlignment,
            state_cfg.numWorlds, state_cfg.numTaskGraphs, state_cfg.numExportedBuffers,
        };
        mb2_compile_config cc {
            compile_cfg.userSources.data(), (uint32_t)compile_cfg.userSources.size(),
            compile_cfg.userCompileFlags.data(), (uint32_t)compile_cfg.userCompileFlags.size(),
            (uint32_t)compile_cfg.optMode,
        };
        mb2_render_config rc {};
        if (render_cfg.has_value()) {
            static_assert(sizeof(render::MeshBVHData) == sizeof(mb2_mesh_bvh_view), "MeshBVHData layout");
            rc.render_mode = (uint32_t)render_cfg->renderMode;
            memcpy(&rc.geo_bvh_data, &render_cfg->geoBVHData, sizeof(rc.geo_bvh_data));
            rc.material_data.textures = (void *)render_cfg->materialData.textures;
            rc.material_data.num_texture_buffers = render_cfg->materialData.numTextureBuffers;
            rc.material_data.texture_buffers = (void *)render_cfg->materialData.textureBuffers;
            rc.material_data.materials = (void *)render_cfg->materialData.materials;
            rc.render_resolution = render_cfg->renderResolution;
            rc.near_plane = render_cfg->nearPlane;
            rc.far_plane = render_cfg->farPlane;
            rc.render_width = image_size.width;
            rc.render_height = image_size.height;
            rc.segmentation = outputs.segmentation ? 1u : 0u;
            rc.normals = outputs.normals ? 1u : 0u;
            rc.projection = (uint32_t)projection;
        }
        int gpu_id = mb2_device_of_context((void *)cu_ctx);
        h_ = mb2_executor_create(&sc, &cc, gpu_id, render_cfg.has_value() ? &rc : nullptr);
        if (!h_) detail::fatal("MWCudaExecutor");
    }

    mb2_executor *h_;
};

}

inline void madrona_b200::ExecutorSnapshot::save(cudaStream_t strm)
{
    if (mb2_snapshot_save(exec_, h_, (void *)strm) != 0) ::madrona::detail::fatal("ExecutorSnapshot::save");
}

inline void madrona_b200::ExecutorSnapshot::restore(cudaStream_t strm)
{
    if (mb2_snapshot_restore(exec_, h_, (void *)strm) != 0) ::madrona::detail::fatal("ExecutorSnapshot::restore");
}
