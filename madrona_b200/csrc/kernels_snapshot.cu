// kernels_snapshot.cu -- executor snapshots: save every byte of device state that a later
// launch can read into a device buffer, and restore it, each as one kernel launch.
//
// The host builds a segment list once per snapshot (DESIGN.md "Snapshots" has the state
// inventory): {live address, snapshot address, bytes per row, row count}.  Counts that only
// the device knows (a table's numRows, numEntitySlots, the arena offsets) are read by the
// kernel through a pointer: a save reads the live count, a restore the count the snapshot
// holds, never the one it is overwriting -- so no block has to wait for another.  A segment
// is cut into fixed-size chunks of its capacity; blocks take chunks in a grid-stride loop
// and a chunk past the segment's live length exits at once.
#include "engine.hpp"
#include "physics_host.hpp"
#include "physics_state.h"
#include "render_state.h"

#include <cstddef>

namespace mb2 {

constexpr int kSnapThreads = 256;
constexpr int kSnapUnitsPerThread = 8;                                             // 16-byte units
constexpr i64 kSnapChunkBytes = (i64)kSnapThreads * kSnapUnitsPerThread * 16;   // 32 KiB
constexpr int kSnapBlocksPerSM = 4;   // resident at 64 registers per thread

enum SnapFlags : u32 {
    // `live` is the device address of the pointer to the live bytes: a table column, whose
    // pointer the sort flips between the column and its twin buffer
    SnapIndirect = 1u,
    SnapCount64 = 2u,   // the row count is a u64 (an arena offset in bytes), else an i32
};

struct alignas(16) SnapSegment {
    u64 live;
    u64 snap;          // in the snapshot buffer
    u64 liveCount;     // device address of the live row count; 0: `rows` rows, always
    u64 snapCount;     // the same count where the snapshot holds it (what a restore reads)
    i64 rows;          // fixed row count, or the most rows the snapshot has room for
    i64 firstChunk;    // chunks of all earlier segments
    u32 rowBytes;
    u32 flags;
    u32 pad[2];
};
static_assert(sizeof(SnapSegment) == 64, "SnapSegment layout");

__device__ __forceinline__ i64 snapRows(const SnapSegment &g, int restore)
{
    const u64 cp = restore ? g.snapCount : g.liveCount;
    if (cp == 0) return g.rows;
    const i64 n = (g.flags & SnapCount64) ? (i64)min(*(const u64 *)cp, (u64)g.rows) : (i64)*(const i32 *)cp;
    return n < 0 ? 0 : min(n, g.rows);
}

// One block copies len <= kSnapChunkBytes bytes: 16-byte units when both ends are 16-byte
// aligned (all 8 loads of a thread issued before its stores), then 4-byte units, then bytes
// (the tails of 12-, 24- or 28-byte rows and unaligned scalars)
__device__ __forceinline__ void snapCopyChunk(const char *__restrict__ src, char *__restrict__ dst, int len)
{
    const int t = threadIdx.x;
    int done = 0;
    if ((((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
        const int n = len >> 4;
        const uint4 *s = (const uint4 *)src;
        uint4 *d = (uint4 *)dst;
        uint4 v[kSnapUnitsPerThread];
#pragma unroll
        for (int k = 0; k < kSnapUnitsPerThread; k++) {
            const int i = t + k * kSnapThreads;
            if (i < n) v[k] = s[i];
        }
#pragma unroll
        for (int k = 0; k < kSnapUnitsPerThread; k++) {
            const int i = t + k * kSnapThreads;
            if (i < n) d[i] = v[k];
        }
        done = n << 4;
    }
    if ((((uintptr_t)(src + done) | (uintptr_t)(dst + done)) & 3) == 0) {
        const int n = (len - done) >> 2;
        const u32 *s = (const u32 *)(src + done);
        u32 *d = (u32 *)(dst + done);
        for (int i = t; i < n; i += kSnapThreads) d[i] = s[i];
        done += n << 2;
    }
    for (int i = done + t; i < len; i += kSnapThreads) dst[i] = src[i];
}

__global__ void __launch_bounds__(kSnapThreads)
snapshotCopyKernel(const SnapSegment *__restrict__ segs, int num_segs, i64 num_chunks, int restore)
{
    for (i64 c = blockIdx.x; c < num_chunks; c += gridDim.x) {
        // the segment of chunk c: the last one that starts at or before it
        int lo = 0, hi = num_segs - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (segs[mid].firstChunk <= c) lo = mid;
            else hi = mid - 1;
        }
        const SnapSegment &g = segs[lo];
        const i64 bytes = snapRows(g, restore) * (i64)g.rowBytes;
        const i64 off = (c - g.firstChunk) * kSnapChunkBytes;
        if (off >= bytes) continue;
        char *live = (g.flags & SnapIndirect) ? *(char *const *)g.live : (char *)g.live;
        char *snap = (char *)g.snap;
        const int len = (int)min(bytes - off, kSnapChunkBytes);
        if (restore) snapCopyChunk(snap + off, live + off, len);
        else snapCopyChunk(live + off, snap + off, len);
    }
}

// ---- host side -----------------------------------------------------------------------

struct Snapshot {
    Executor *owner = nullptr;
    std::vector<SnapSegment> plan;       // snap / snapCount: offsets into the buffer
    std::vector<SnapSegment> uploaded;   // the plan with device addresses (source of the last upload)
    std::vector<int64_t> capacities;     // what the plan was sized for (capacitySignature)
    SnapSegment *dSegs = nullptr;
    size_t segCapacity = 0;
    char *buf = nullptr;
    int64_t bytes = 0;
    int64_t numChunks = 0;
    bool saved = false;
};

// Table, entity store and instance-list capacities: host-known, they only grow (between
// steps, growTablesFromStatus)
static std::vector<int64_t> capacitySignature(Executor *ex)
{
    const EngineState &S = *ex->hState;
    std::vector<int64_t> sig;
    for (uint32_t a = 0; a < S.numArchetypes; a++) sig.push_back(S.tables[a].capacity);
    sig.push_back(S.entityCapacity);
    const RenderState *R = renderHostState(ex);
    sig.push_back(R ? R->instanceCapacity : 0);
    return sig;
}

namespace {

struct Planner {
    std::vector<SnapSegment> segs;
    int64_t offset = 0;
    int64_t chunks = 0;

    // returns the segment's offset in the snapshot buffer
    int64_t add(const void *live, u32 flags, int64_t rows, uint64_t row_bytes,
                const void *live_count = nullptr, int64_t snap_count = -1)
    {
        const int64_t bytes = rows * (int64_t)row_bytes;
        if (!live || bytes <= 0) return -1;
        const int64_t align = bytes >= 256 ? 256 : 16;
        offset = (offset + align - 1) / align * align;
        SnapSegment g {};
        g.live = (u64)(uintptr_t)live;
        g.snap = (u64)offset;
        g.liveCount = (u64)(uintptr_t)live_count;
        g.snapCount = snap_count < 0 ? 0 : (u64)snap_count;
        g.rows = rows;
        g.firstChunk = chunks;
        g.rowBytes = (u32)row_bytes;
        g.flags = flags;
        segs.push_back(g);
        const int64_t at = offset;
        offset += bytes;
        chunks += (bytes + kSnapChunkBytes - 1) / kSnapChunkBytes;
        return at;
    }
    int64_t scalar(const void *live, uint64_t bytes) { return add(live, 0, 1, bytes); }
};

}

static_assert(offsetof(EngineState, errorArchetype) == offsetof(EngineState, errorFlags) + 4, "errorFlags");
static_assert(offsetof(EngineState, freeHead) == offsetof(EngineState, numEntitySlots) + 4, "freeHead");
static_assert(offsetof(TableDesc, highWater) == offsetof(TableDesc, needsSort) + 8, "TableDesc flags");
static_assert(offsetof(RenderState, totalNumInstances) == offsetof(RenderState, totalNumViews) + 4, "totals");

// The state inventory (DESIGN.md "Snapshots"): scalars first, so that every count a bulk
// segment reads has its place in the snapshot already
static void buildPlan(Executor *ex, Planner *p)
{
    const EngineState &S = *ex->hState;
    EngineState *d = ex->dState;
    const int64_t W = S.numWorlds;

    p->scalar(&d->errorFlags, 8);                                   // + errorArchetype
    const int64_t ent_at = p->scalar(&d->numEntitySlots, 12);       // + freeHead
    const int64_t tmp_at = p->scalar(&d->tmpOffset, 8);
    const int64_t persist_at = p->scalar(&d->persistOffset, 8);
    int64_t rows_at[kMaxArchetypes];
    for (uint32_t a = 0; a < S.numArchetypes; a++) {
        rows_at[a] = -1;
        if (!S.archetypes[a].registered) continue;
        rows_at[a] = p->scalar(&d->tables[a].numRows, 4);
        p->scalar(&d->tables[a].needsSort, 12);                     // + isSingleton, highWater
    }
    if (S.physics) p->scalar(&S.physics->hasSpherePrims, 4);
    const RenderState *R = renderHostState(ex);
    int64_t totals_at = -1;
    if (R) totals_at = p->scalar(&S.render->totalNumViews, 8);     // + totalNumInstances

    // tables: live rows of every column, per-world offsets and counts
    for (uint32_t a = 0; a < S.numArchetypes; a++) {
        if (rows_at[a] < 0) continue;
        const TableDesc &t = S.tables[a];
        for (int32_t c = 0; c < t.numColumns; c++) {
            p->add(&d->tables[a].columns[c], SnapIndirect, t.capacity, t.columnBytes[c],
                   &d->tables[a].numRows, rows_at[a]);
        }
        p->add(t.worldOffsets, 0, W, sizeof(i32));
        p->add(t.worldCounts, 0, W, sizeof(i32));
    }
    // entity store
    p->add(S.entitySlots, 0, S.entityCapacity, sizeof(EntitySlot), &d->numEntitySlots, ent_at);
    p->add(S.idCaches, 0, W, sizeof(IDCache));
    // world data, arenas, custom node data
    p->add(S.worldData, 0, W, S.worldDataStride);
    p->add(S.tmpArena, SnapCount64, (int64_t)S.tmpCapacity, 1, &d->tmpOffset, tmp_at);
    p->add(S.persistArena, SnapCount64, (int64_t)S.persistCapacity, 1, &d->persistOffset, persist_at);
    p->add(S.nodeData, 0, std::min<int64_t>(S.numNodeDatas, kMaxNodeDatas + 1), kNodeDataBytes);
    // what the render graph reads from the last render-prepare: views, the instance list
    // and TLAS (world w's at instanceOffsets[w], all within the first totalNumInstances
    // rows), lights
    if (R) {
        const int64_t inst_at = totals_at + 4;
        p->add(R->views, 0, R->maxViews, sizeof(RenderView), &d->tables[R->outputArchetype].numRows,
               rows_at[R->outputArchetype]);
        p->add(R->instances, 0, R->instanceCapacity, sizeof(RenderInstance), &S.render->totalNumInstances, inst_at);
        p->add(R->tlasNodes, 0, R->instanceCapacity, sizeof(QBVHNode), &S.render->totalNumInstances, inst_at);
        p->add(R->instanceCounts, 0, W, sizeof(i32));
        p->add(R->instanceOffsets, 0, W, sizeof(i32));
        p->add(R->tlasNodeCounts, 0, W, sizeof(i32));
        p->add(R->tlasDepths, 0, W, sizeof(i32));
        p->add(R->lights, 0, W * kMaxLightsPerWorld, sizeof(RenderLight));
        p->add(R->lightCounts, 0, W, sizeof(i32));
    }
}

// (re)size the snapshot for the executor's current capacities and upload its segment list
static bool snapshotPlan(Snapshot *s, cudaStream_t st, std::string *err)
{
    Executor *ex = s->owner;
    Planner p;
    buildPlan(ex, &p);
    const int64_t bytes = std::max<int64_t>(p.offset, 16);
    auto fail = [&](const char *what, cudaError_t e) {
        *err = std::string("snapshot: ") + what + ": " + cudaGetErrorString(e);
        return false;
    };
    cudaError_t e;
    if (bytes > s->bytes) {
        if (s->buf && (e = cudaFreeAsync(s->buf, st)) != cudaSuccess) return fail("cudaFreeAsync", e);
        s->buf = nullptr;
        s->bytes = 0;
        if ((e = cudaMallocAsync((void **)&s->buf, (size_t)bytes, st)) != cudaSuccess) {
            s->buf = nullptr;
            return fail("cudaMallocAsync", e);
        }
        s->bytes = bytes;
    }
    if (p.segs.size() > s->segCapacity) {
        if (s->dSegs && (e = cudaFreeAsync(s->dSegs, st)) != cudaSuccess) return fail("cudaFreeAsync", e);
        s->dSegs = nullptr;
        s->segCapacity = 0;
        if ((e = cudaMallocAsync((void **)&s->dSegs, sizeof(SnapSegment) * p.segs.size(), st)) != cudaSuccess) {
            s->dSegs = nullptr;
            return fail("cudaMallocAsync", e);
        }
        s->segCapacity = p.segs.size();
    }
    s->plan = p.segs;
    s->uploaded = p.segs;
    const u64 base = (u64)(uintptr_t)s->buf;
    for (SnapSegment &g : s->uploaded) {
        g.snap += base;
        if (g.liveCount) g.snapCount += base;
    }
    if (!s->uploaded.empty() &&
            (e = cudaMemcpyAsync(s->dSegs, s->uploaded.data(), sizeof(SnapSegment) * s->uploaded.size(),
                                 cudaMemcpyHostToDevice, st)) != cudaSuccess) {
        return fail("segment list upload", e);
    }
    s->numChunks = p.chunks;
    s->capacities = capacitySignature(ex);
    s->saved = false;
    return true;
}

static bool snapshotLaunch(Snapshot *s, cudaStream_t st, int restore, std::string *err)
{
    if (s->numChunks == 0 || s->uploaded.empty()) return true;
    const int64_t grid = std::max<int64_t>(1, std::min<int64_t>(s->numChunks,
                                                                (int64_t)s->owner->numSMs * kSnapBlocksPerSM));
    snapshotCopyKernel<<<(unsigned)grid, kSnapThreads, 0, st>>>(s->dSegs, (int)s->uploaded.size(), s->numChunks,
                                                                restore);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        *err = std::string(restore ? "snapshot restore" : "snapshot save") + ": " + cudaGetErrorString(e);
        return false;
    }
    return true;
}

Snapshot *snapshotCreate(Executor *ex, std::string *err)
{
    cudaSetDevice(ex->gpu);
    Snapshot *s = new Snapshot();
    s->owner = ex;
    if (!snapshotPlan(s, ex->stream, err)) {
        snapshotDestroy(s);
        return nullptr;
    }
    const cudaError_t e = cudaStreamSynchronize(ex->stream);
    if (e != cudaSuccess) {
        *err = std::string("snapshot: ") + cudaGetErrorString(e);
        snapshotDestroy(s);
        return nullptr;
    }
    return s;
}

bool snapshotSave(Snapshot *s, cudaStream_t st, std::string *err)
{
    cudaSetDevice(s->owner->gpu);
    // a table (and with it the entity store and the instance list) grew since the plan
    // was made: more rows may be live than the snapshot has room for
    if (capacitySignature(s->owner) != s->capacities && !snapshotPlan(s, st, err)) return false;
    if (!snapshotLaunch(s, st, 0, err)) return false;
    s->saved = true;
    return true;
}

bool snapshotRestore(Snapshot *s, cudaStream_t st, std::string *err)
{
    if (!s->saved) {
        *err = "snapshot restore: the snapshot was never saved";
        return false;
    }
    cudaSetDevice(s->owner->gpu);
    // capacities never shrink, so the plan of the last save fits the live state as it is now
    return snapshotLaunch(s, st, 1, err);
}

int64_t snapshotBytes(const Snapshot *s) { return s->bytes; }

// Bytes the last save copied: the plan's rows at the counts the snapshot holds (waits for the device)
int64_t snapshotSavedBytes(Snapshot *s)
{
    if (!s->saved) return 0;
    cudaSetDevice(s->owner->gpu);
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    int64_t total = 0;
    for (const SnapSegment &g : s->uploaded) {
        int64_t rows = g.rows;
        if (g.liveCount) {
            if (g.flags & SnapCount64) {
                u64 n = 0;
                if (cudaMemcpy(&n, (const void *)g.snapCount, sizeof(n), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
                rows = (int64_t)std::min<u64>(n, (u64)g.rows);
            } else {
                i32 n = 0;
                if (cudaMemcpy(&n, (const void *)g.snapCount, sizeof(n), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
                rows = std::max<int64_t>(0, std::min<int64_t>(n, g.rows));
            }
        }
        total += rows * (int64_t)g.rowBytes;
    }
    return total;
}

Executor *snapshotOwner(const Snapshot *s) { return s->owner; }

void snapshotDestroy(Snapshot *s)
{
    if (!s) return;
    cudaSetDevice(s->owner->gpu);
    // a save or restore may still be queued on any stream: wait for the device, as the
    // executor's own cudaFree calls do (cudaFree does not wait for stream-ordered allocations)
    if (s->buf || s->dSegs) cudaDeviceSynchronize();
    if (s->buf) cudaFree(s->buf);
    if (s->dSegs) cudaFree(s->dSegs);
    delete s;
}

}
