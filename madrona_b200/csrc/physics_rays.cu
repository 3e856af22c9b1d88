// physics_rays.cu -- mb2_trace_physics_rays: batches of rays from device memory against the
// worlds' broadphase trees, each ray answered as broadphase::BVH::traceRay answers it in its
// world (physics_ray.h, the code both compile; this TU, like the simulator, without FMA
// contraction).
//
// Rays come in any world order, with repeats.  They are grouped by world on the device with a
// counting pass -- per-world histogram, one-block scan, scatter of ray indices into slots -- so
// the rays of one world sit in consecutive slots and are traced where the world's boxes are
// shared:
//   * worlds of up to kSmallWorldLeaves leaves: one lane per slot.  A warp's lanes are mostly
//     rays of one world and read the same ordered box at the same time (a broadcast load);
//   * larger worlds (MADRONA_B200_MAX_BODIES_PER_WORLD > 128): one block per world stages the
//     world's orderedBoxes (32 B per leaf, at most 128 KB) in shared memory once, for all of
//     that world's rays.
// Every launch goes on the caller's stream; nothing synchronizes the host.
#include "physics_host.hpp"
#include "physics_state.h"
#include "physics_ray.h"

#include <algorithm>

namespace mb2 {

using madrona::math::Vector3;

constexpr int kRayThreads = 256;          // count, scatter and small-world trace kernels
constexpr int kRayScanThreads = 1024;
constexpr int kRayLargeThreads = 256;
constexpr i32 kSmallWorldLeaves = kMinWorldBodiesCap;

struct PhysicsRayHost {
    i32 *counts = nullptr;       // [numWorlds]: rays per world, then the scatter's cursors
    i32 *offsets = nullptr;      // [numWorlds + 1]: first slot of each world's rays
    u32 *order = nullptr;        // [capacity]: slot -> ray index
    u32 capacity = 0;
    unsigned largeBlocks = 0;    // resident blocks of physRaysTraceLargeKernel (0: not queried yet)
};

struct RayJob {
    const i32 *world;
    const float *origin;
    const float *direction;
    const float *maxT;           // null: +inf
    i32 *entity;                 // [n][2] {gen, id}, or null
    float *t;
    float *normal;               // [n][3], or null
    u32 n;
    i32 *counts;
    i32 *offsets;
    u32 *order;
    i32 maxStaged;               // leaves physRaysTraceLargeKernel's shared memory holds
};

__device__ __forceinline__ const WorldBVH &rayWorldBVH(const EngineState &S, i32 w)
{
    return ((const WorldBVH *)S.tables[S.physics->bvhArchetype].columns[2])[w];
}

// hit: the leaf's entity, t and world-frame normal; miss (leaf < 0): Entity::none(), 0, (0, 0, 0)
__device__ __forceinline__ void writeRayResult(const RayJob &J, const WorldBVH *bvh, u32 i, i32 leaf, float t,
                                               Vector3 normal)
{
    u32 gen = 0xFFFFFFFFu;
    i32 id = -1;
    if (leaf >= 0) {
        const u64 e = bvh->leafEntities[leaf];
        gen = (u32)(e & 0xFFFFFFFFull);
        id = (i32)(u32)(e >> 32);
    } else {
        t = 0.f;
        normal = Vector3 { 0, 0, 0 };
    }
    if (J.entity) {
        J.entity[2 * i] = (i32)gen;
        J.entity[2 * i + 1] = id;
    }
    if (J.t) J.t[i] = t;
    if (J.normal) {
        J.normal[3 * i] = normal.x;
        J.normal[3 * i + 1] = normal.y;
        J.normal[3 * i + 2] = normal.z;
    }
}

__device__ __forceinline__ bool rayWorldValid(const EngineState &S, i32 w)
{
    return w >= 0 && (u32)w < S.numWorlds;
}

// per-world histogram; a ray of a world outside [0, numWorlds) is answered here with a miss and
// raises ErrPhysicsRayWorld
__global__ void __launch_bounds__(kRayThreads)
physRaysCountKernel(EngineState *Sp, RayJob J)
{
    EngineState &S = *Sp;
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= J.n) return;
    const i32 w = J.world[i];
    if (rayWorldValid(S, w)) {
        atomicAdd(&J.counts[w], 1);
    } else {
        writeRayResult(J, nullptr, i, -1, 0.f, Vector3 { 0, 0, 0 });
        atomicOr(&S.errorFlags, (u32)ErrPhysicsRayWorld);
    }
}

// 1 block: exclusive scan of counts -> offsets[0 .. numWorlds]; counts become the scatter's cursors
__global__ void __launch_bounds__(kRayScanThreads)
physRaysScanKernel(const EngineState *Sp, RayJob J)
{
    const i32 W = (i32)Sp->numWorlds;
    const i32 per = (W + kRayScanThreads - 1) / kRayScanThreads;
    const i32 first = min(W, (i32)threadIdx.x * per), last = min(W, first + per);
    i32 sum = 0;
    for (i32 w = first; w < last; w++) sum += J.counts[w];

    __shared__ i32 warp_incl[kRayScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    i32 incl = sum;
    for (int o = 1; o < 32; o <<= 1) {
        const i32 up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
    }
    if (lane == 31) warp_incl[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        i32 v = warp_incl[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const i32 up = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += up;
        }
        warp_incl[lane] = v;
    }
    __syncthreads();
    i32 off = incl - sum + (warp > 0 ? warp_incl[warp - 1] : 0);
    for (i32 w = first; w < last; w++) {
        const i32 c = J.counts[w];
        J.offsets[w] = off;
        J.counts[w] = off;
        off += c;
    }
    if (threadIdx.x == 0) J.offsets[W] = warp_incl[kRayScanThreads / 32 - 1];
}

__global__ void __launch_bounds__(kRayThreads)
physRaysScatterKernel(const EngineState *Sp, RayJob J)
{
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= J.n) return;
    const i32 w = J.world[i];
    if (!rayWorldValid(*Sp, w)) return;
    J.order[atomicAdd(&J.counts[w], 1)] = i;
}

__device__ __forceinline__ void loadRay(const RayJob &J, u32 i, Vector3 *o, Vector3 *d, float *t_max)
{
    *o = Vector3 { J.origin[3 * i], J.origin[3 * i + 1], J.origin[3 * i + 2] };
    *d = Vector3 { J.direction[3 * i], J.direction[3 * i + 1], J.direction[3 * i + 2] };
    *t_max = J.maxT ? J.maxT[i] : __int_as_float(0x7f800000);
}

// One lane per slot, for the rays of worlds of up to kSmallWorldLeaves leaves (all worlds when
// `large` is false); the other slots are left to physRaysTraceLargeKernel.
__global__ void __launch_bounds__(kRayThreads)
physRaysTraceKernel(const EngineState *Sp, RayJob J, bool large)
{
    const EngineState &S = *Sp;
    const u32 slot = blockIdx.x * blockDim.x + threadIdx.x;
    const WorldBVH *bvh = nullptr;
    u32 i = 0;
    if (slot < (u32)J.offsets[S.numWorlds]) {
        i = J.order[slot];
        bvh = &rayWorldBVH(S, J.world[i]);
        if (large && bvh->numTraversal > kSmallWorldLeaves) bvh = nullptr;
    }
    const unsigned peers = __ballot_sync(0xffffffffu, bvh != nullptr);
    if (!bvh) return;
    Vector3 o, d, normal;
    float t_max, t;
    loadRay(J, i, &o, &d, &t_max);
    const i32 leaf = physray::traceWorld(*bvh, bvh->orderedBoxes, bvh->numTraversal, peers, o, d, t_max, &t, &normal);
    writeRayResult(J, bvh, i, leaf, t, normal);
}

// A persistent grid over the worlds; a world of more than kSmallWorldLeaves leaves with rays
// gets the block: its orderedBoxes are staged in shared memory, then the block's threads take
// its rays in turn.
__global__ void __launch_bounds__(kRayLargeThreads)
physRaysTraceLargeKernel(const EngineState *Sp, RayJob J)
{
    extern __shared__ float4 ray_stage[];
    const EngineState &S = *Sp;
    for (i32 w = blockIdx.x; w < (i32)S.numWorlds; w += gridDim.x) {
        const WorldBVH &bvh = rayWorldBVH(S, w);
        const i32 num_boxes = bvh.numTraversal;
        const i32 first = J.offsets[w], count = J.offsets[w + 1] - first;
        if (count == 0 || num_boxes <= kSmallWorldLeaves) continue;
        const float4 *src = reinterpret_cast<const float4 *>(bvh.orderedBoxes);
        const i32 staged = num_boxes <= J.maxStaged ? num_boxes : 0;
        for (i32 k = threadIdx.x; k < 2 * staged; k += blockDim.x) ray_stage[k] = src[k];
        __syncthreads();
        // (a world past the knob, which its step refuses, is traced from global memory)
        const PVec4 *boxes = num_boxes <= J.maxStaged ? reinterpret_cast<const PVec4 *>(ray_stage) : bvh.orderedBoxes;
        for (i32 base = 0; base < count; base += blockDim.x) {
            const i32 r = base + (i32)threadIdx.x;
            const unsigned peers = __ballot_sync(0xffffffffu, r < count);
            if (r < count) {
                const u32 i = J.order[first + r];
                Vector3 o, d, normal;
                float t_max, t;
                loadRay(J, i, &o, &d, &t_max);
                const i32 leaf = physray::traceWorld(bvh, boxes, num_boxes, peers, o, d, t_max, &t, &normal);
                writeRayResult(J, &bvh, i, leaf, t, normal);
            }
        }
        __syncthreads();     // every thread is done with the stage before the next world's
    }
}

static size_t largeRayStageBytes(const PhysicsState &P)
{
    return (size_t)P.maxWorldBodies * 2 * sizeof(PVec4);
}

// The kernel's dynamic shared memory limit belongs to the function on the device, not to an
// executor: set it for this executor's stage before every launch, since another executor on the
// device may have set it for a smaller MADRONA_B200_MAX_BODIES_PER_WORLD since.
static bool setLargeRayStage(const PhysicsState &P)
{
    return cudaFuncSetAttribute(physRaysTraceLargeKernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)largeRayStageBytes(P)) == cudaSuccess;
}

static bool misaligned(const void *p)
{
    return ((uintptr_t)p & 3u) != 0;
}

bool physicsTraceRays(Executor *ex, const mb2_physics_rays &rays, uint32_t n, const mb2_physics_ray_hits &hits,
                      cudaStream_t s, std::string *err)
{
    const PhysicsState *P = physicsHostState(ex);
    if (!P) {
        *err = "the simulator never called PhysicsSystem::registerTypes: there is no physics scene to query";
        return false;
    }
    if (n == 0) return true;
    if (!rays.world || !rays.origin || !rays.direction) {
        *err = "rays: world, origin and direction must not be NULL";
        return false;
    }
    if (!hits.entity && !hits.t && !hits.normal) {
        *err = "every output (entity, t, normal) is NULL";
        return false;
    }
    const void *ptrs[] = { rays.world, rays.origin, rays.direction, rays.max_t, hits.entity, hits.t, hits.normal };
    const char *names[] = { "world", "origin", "direction", "max_t", "entity", "t", "normal" };
    for (int k = 0; k < 7; k++) {
        if (misaligned(ptrs[k])) {
            *err = std::string(names[k]) + " is not 4-byte aligned";
            return false;
        }
    }

    cudaSetDevice(ex->gpu);
    const u32 W = ex->hState->numWorlds;
    const bool large = P->maxWorldBodies > kSmallWorldLeaves;
    PhysicsRayHost *rh = ex->physicsRays;
    if (!rh) {
        rh = new PhysicsRayHost();
        ex->physicsRays = rh;
        if (cudaMalloc((void **)&rh->counts, sizeof(i32) * (2 * (size_t)W + 1)) != cudaSuccess) {
            rh->counts = nullptr;
            *err = "ray query scratch allocation failed";
            return false;
        }
        rh->offsets = rh->counts + W;
        if (large) {
            int per_sm = 0;
            if (!setLargeRayStage(*P) ||
                cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, physRaysTraceLargeKernel, kRayLargeThreads,
                                                              largeRayStageBytes(*P)) != cudaSuccess) {
                cudaGetLastError();
                per_sm = 0;
            }
            rh->largeBlocks = (unsigned)ex->numSMs * (unsigned)per_sm;
        }
    }
    if (!rh->counts) {
        *err = "ray query scratch allocation failed";
        return false;
    }
    if (large && (rh->largeBlocks == 0 || !setLargeRayStage(*P))) {
        cudaGetLastError();
        *err = "the large-world ray kernel's shared memory (MADRONA_B200_MAX_BODIES_PER_WORLD) does not fit the device";
        return false;
    }
    // the slot list only grows; cudaFree waits for the device, so no earlier call still reads it
    if (n > rh->capacity) {
        const u32 cap = std::max(n, std::min(2 * rh->capacity, 0x7fffffffu));
        if (rh->order) cudaFree(rh->order);
        rh->order = nullptr;
        rh->capacity = 0;
        if (cudaMalloc((void **)&rh->order, sizeof(u32) * (size_t)cap) != cudaSuccess) {
            rh->order = nullptr;
            *err = "ray query scratch allocation failed";
            return false;
        }
        rh->capacity = cap;
    }

    RayJob J;
    J.world = rays.world;
    J.origin = rays.origin;
    J.direction = rays.direction;
    J.maxT = rays.max_t;
    J.entity = (i32 *)hits.entity;
    J.t = hits.t;
    J.normal = hits.normal;
    J.n = n;
    J.counts = rh->counts;
    J.offsets = rh->offsets;
    J.order = rh->order;
    J.maxStaged = P->maxWorldBodies;
    const unsigned grid = (n + kRayThreads - 1) / kRayThreads;
    cudaMemsetAsync(rh->counts, 0, sizeof(i32) * W, s);
    physRaysCountKernel<<<grid, kRayThreads, 0, s>>>(ex->dState, J);
    physRaysScanKernel<<<1, kRayScanThreads, 0, s>>>(ex->dState, J);
    physRaysScatterKernel<<<grid, kRayThreads, 0, s>>>(ex->dState, J);
    physRaysTraceKernel<<<grid, kRayThreads, 0, s>>>(ex->dState, J, large);
    if (large) {
        physRaysTraceLargeKernel<<<std::min(rh->largeBlocks, W), kRayLargeThreads, largeRayStageBytes(*P), s>>>(
            ex->dState, J);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        *err = std::string("launch failed: ") + cudaGetErrorString(e);
        return false;
    }
    return true;
}

void physicsRaysDestroy(Executor *ex)
{
    PhysicsRayHost *rh = ex->physicsRays;
    if (!rh) return;
    if (rh->counts) cudaFree(rh->counts);
    if (rh->order) cudaFree(rh->order);
    delete rh;
    ex->physicsRays = nullptr;
}

}
