// Host hooks for the engine-owned systems (rigid-body physics, ray-cast
// renderer): kernels_physics.cu / kernels_render.cu.
#pragma once
#include "engine.hpp"
#include "../../include/madrona_b200.h"

namespace mb2 {

// MADRONA_B200_MAX_HULL_SIZE (16 when unset), or false and why its value is invalid
bool physicsMaxHullSize(int *size, std::string *err);
// MADRONA_B200_MAX_BODIES_PER_WORLD (128 when unset), or false and why its value is invalid
bool physicsMaxWorldBodies(int *bodies, std::string *err);
bool physicsHostCreate(Executor *ex, std::string *err);
bool physicsHostAfterRegistry(Executor *ex, const mb2_render_config *rc, std::string *err);
void physicsHostDestroy(Executor *ex);
// reads device-side facts that select kernel variants; call before stream capture begins
void physicsBeforeGraphCapture(Executor *ex);
bool physicsEnqueueNodes(Executor *ex, const NodeRecord *recs, uint32_t count, cudaStream_t s,
                         std::string *err);
LaunchGraph *physicsBuildRenderGraph(Executor *ex, std::string *err);
// batch ray-cast renderer (kernels_render.cu)
// the image size of a render config, or false and why the config is invalid
bool renderImageSize(const mb2_render_config *rc, uint32_t *width, uint32_t *height, std::string *err);
// whether a render config asks for the segmentation output, or false and why it is invalid
bool renderSegmentation(const mb2_render_config *rc, uint32_t *on, std::string *err);
// the camera model of a render config (0 pinhole, 1 panorama), or false and why it is invalid
bool renderProjection(const mb2_render_config *rc, uint32_t *projection, std::string *err);
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
// algorithmic bytes of one launch of a physics node + a short name (profiling)
uint64_t physicsNodeBytes(Executor *ex, const NodeRecord &rec, const char **name, int64_t *rows);

}
