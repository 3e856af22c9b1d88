// Host hooks for the engine-owned systems (rigid-body physics, ray-cast
// renderer): kernels_physics.cu / kernels_render.cu.
#pragma once
#include "engine.hpp"
#include "../../include/madrona_b200.h"

namespace mb2 {

struct PhysicsState;

bool physicsHostCreate(Executor *ex, std::string *err);
bool physicsHostAfterRegistry(Executor *ex, std::string *err);
void physicsHostDestroy(Executor *ex);
// reads device-side facts that select kernel variants; call before stream capture begins
void physicsBeforeGraphCapture(Executor *ex);
bool physicsEnqueueNodes(Executor *ex, const NodeRecord *recs, uint32_t count, cudaStream_t s,
                         std::string *err);
LaunchGraph *physicsBuildRenderGraph(Executor *ex, std::string *err);
// batch ray-cast renderer (kernels_render.cu)
// the image size, outputs and projection a render config (or null) asks for, or false and why
// the config is invalid
bool renderParseConfig(const mb2_render_config *rc, RenderSettings *out, std::string *err);
bool renderHostCreate(Executor *ex, const mb2_render_config *rc, std::string *err);
bool renderHostAfterRegistry(Executor *ex, std::string *err);
void renderHostDestroy(Executor *ex);
bool renderEnqueuePrepare(Executor *ex, cudaStream_t s, std::string *err);
// after a renderable table grew: map instance-list rows for its new capacity
bool renderEnsureCapacity(Executor *ex, std::string *err);
void *renderDebugHitBuffer(Executor *ex);
void *renderDebugBuffer(Executor *ex, int which);
uint64_t renderBytesPerFrame(Executor *ex, int64_t num_views);
// host copy of the ray caster's state (device pointers, capacities), null when it is not active
const RenderState *renderHostState(Executor *ex);
// mb2_render_free_views after its null checks: checks the rest before any CUDA call, then
// enqueues the views' copy, their conversion, the ray caster and the status copy on s
bool renderFreeViews(Executor *ex, const mb2_free_view *views, uint32_t num_views, uint32_t width,
                     uint32_t height, uint32_t projection, const mb2_free_view_outputs &outputs, cudaStream_t s,
                     std::string *err);
// device records -> RenderView (render_free_views.cu, compiled without FMA contraction)
struct RenderView;
void renderConvertFreeViews(const mb2_free_view *in, RenderView *out, uint32_t n, cudaStream_t s);
// host copy of the physics state (device pointers, knobs), null when the simulator never called
// PhysicsSystem::registerTypes
const PhysicsState *physicsHostState(Executor *ex);
// mb2_trace_physics_rays after its null checks: checks the rest before any CUDA call, then
// enqueues the grouping of the rays by world and their traces on s (physics_rays.cu)
bool physicsTraceRays(Executor *ex, const mb2_physics_rays &rays, uint32_t n, const mb2_physics_ray_hits &hits,
                      cudaStream_t s, std::string *err);
void physicsRaysDestroy(Executor *ex);
// algorithmic bytes of one launch of a physics node + a short name (profiling)
uint64_t physicsNodeBytes(Executor *ex, const NodeRecord &rec, const char **name, int64_t *rows);

}
