// engine.hpp -- host-side executor state behind the C ABI (include/madrona_b200.h).
#pragma once

#include <cuda_runtime.h>
#include <cstdint>
#include <string>
#include <vector>

#include "mb2_state.h"
#include "jit.hpp"
#include "vm_alloc.hpp"

namespace mb2 {

struct SortScratch;   // kernels_sort.cu
struct PhysicsHost;   // kernels_physics.cu
struct RenderHost;    // kernels_render.cu
struct PhysicsRayHost;   // physics_rays.cu

// The MADRONA_B200_* environment variables that configure an executor, as parseKnobs read them
struct Knobs {
    uint64_t rowsPerWorld;             // ROWS_PER_WORLD: initial rows per world of a dynamic table
    uint64_t tmpBytes, persistBytes;   // TMP_BYTES, PERSIST_BYTES: the two arenas
    uint64_t maxCandidatesPerWorld;    // MAX_CANDIDATES_PER_WORLD
    uint64_t maxContactsPerWorld;      // MAX_CONTACTS_PER_WORLD
    uint64_t maxHullSize;              // MAX_HULL_SIZE
    uint64_t maxWorldBodies;           // MAX_BODIES_PER_WORLD
    bool tableGrowth;                  // TABLE_GROWTH
    bool graphBranches;                // GRAPH_BRANCHES
    bool fastMath;                     // FAST_MATH
    bool noKernelCache;                // NO_KERNEL_CACHE
    bool renderDebug;                  // RENDER_DEBUG
    std::string kernelCacheDir;        // KERNEL_CACHE_DIR
};

// Reads every knob from the environment (num_worlds sizes the persistent arena's default).
// False, and in *err the knob, what it accepts and what it got, on the first malformed value.
bool parseKnobs(uint32_t num_worlds, Knobs *k, std::string *err);

// What an executor's render config asks of the ray caster (all 0 without one)
struct RenderSettings {
    uint32_t width = 0, height = 0;
    uint32_t segmentation = 0;   // 1: the per-pixel entity id output
    uint32_t projection = 0;     // 0 pinhole, 1 panorama
    uint32_t normals = 0;        // 1: the per-pixel surface normal output
};

struct Executor {
    int gpu = 0;
    int numSMs = 132;
    cudaStream_t stream = nullptr;

    JitModule jit;
    cudaLibrary_t lib = nullptr;
    cudaKernel_t initECS = nullptr, initWorlds = nullptr, initTasks = nullptr;
    std::vector<cudaKernel_t> nodeKernels;
    std::vector<uint64_t> nodeMetaAddrs;
    std::vector<uint32_t> nodeKernelGrid;   // resident blocks of each node kernel (0: not queried yet)

    EngineState *dState = nullptr;     // device
    EngineState *hState = nullptr;     // host mirror (registry, nodes, table descs)
    uint32_t *hStatus = nullptr;       // pinned: [0] errorFlags, [1] errorArchetype

    std::vector<void *> allocations;   // cudaMalloc'd blocks owned by the executor
    void *exported[kMaxExports] = {};
    uint32_t exportArchetype[kMaxExports] = {};
    uint32_t exportRowBytes[kMaxExports] = {};

    SortScratch *sortScratch = nullptr;
    PhysicsHost *physics = nullptr;
    RenderHost *render = nullptr;
    PhysicsRayHost *physicsRays = nullptr;   // scratch of mb2_trace_physics_rays, made by its first call

    Knobs knobs;                     // read and checked before any CUDA call
    RenderSettings renderSettings;   // likewise, from the render config

    // ---- growable storage (vm_alloc.hpp): dynamic archetypes' columns and their sort
    // twins, the sort's key / index / look-back scratch and the entity store keep their
    // base address and get more physical memory between steps (unless knobs.tableGrowth is off)
    std::vector<VMRange> columnRanges[kMaxArchetypes];         // [archetype][column]; empty: fixed table
    std::vector<VMRange> twinRanges[kMaxArchetypes];
    int64_t maxRows[kMaxArchetypes] = {};                      // most rows a table can grow to
    VMRange entityRange;
    int64_t growthEvents = 0;
};

// status block published by the last kernel of every launch graph (pinned host memory)
constexpr int kStatusWords = 2 + kMaxArchetypes;   // errorFlags, errorArchetype, peak rows per table

struct LaunchGraph {
    Executor *owner = nullptr;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    int64_t numKernels = 0;
    int64_t numBranches = 1;   // capture streams used (parallel branches of independent nodes)
    std::string name;
};

void setError(const std::string &msg);

// ---- ahead-of-time engine kernels (kernels_core.cu / kernels_sort.cu) -----
void launchClearTmp(Executor *ex, uint32_t archetype, cudaStream_t s);
void launchResetTmpAlloc(Executor *ex, cudaStream_t s);
void launchLatchNodeCount(Executor *ex, uint32_t node, cudaStream_t s);
void launchStatusCopy(Executor *ex, cudaStream_t s);
void launchFillSingletons(Executor *ex, cudaStream_t s);

bool sortScratchCreate(Executor *ex, std::string *err);
void sortScratchDestroy(Executor *ex);
// Stable sort of `archetype` by the low bits of column `col`; col==1 (WorldID)
// additionally drops rows with key -1 and rebuilds worldOffsets/worldCounts.
void launchSortArchetype(Executor *ex, uint32_t archetype, int32_t col, cudaStream_t s);
int sortNumPasses(Executor *ex, int32_t col);
// the sort's key / index / look-back scratch must cover the largest table
bool sortScratchEnsure(Executor *ex, int32_t max_rows, std::string *err);
// grow a dynamic table to new_capacity rows (columns, twins, entity store, sort scratch)
bool growTable(Executor *ex, uint32_t archetype, int64_t new_capacity, std::string *err);

// ---- snapshots of the device state (kernels_snapshot.cu) -----------------------------
struct Snapshot;
Snapshot *snapshotCreate(Executor *ex, std::string *err);
// one launch on `s` each; save first enlarges the snapshot if a table grew since
bool snapshotSave(Snapshot *snap, cudaStream_t s, std::string *err);
bool snapshotRestore(Snapshot *snap, cudaStream_t s, std::string *err);
int64_t snapshotBytes(const Snapshot *snap);
int64_t snapshotSavedBytes(Snapshot *snap);
Executor *snapshotOwner(const Snapshot *snap);
void snapshotDestroy(Snapshot *snap);

}
