// Device-side ECS runtime for simulator code compiled by NVRTC.
//
// Replaces the reference's GPU StateManager (src/mw/device/state.cpp:163-628,
// src/mw/device/include/madrona/state.{hpp,inl}).  Differences by design:
//   * storage is described by a plain mb2::EngineState block (mb2_state.h) that
//     the ahead-of-time engine kernels (sort, physics, render) share;
//   * component -> column resolution is a dense [archetype][component] i16
//     table instead of a per-archetype perfect hash;
//   * row append is warp-aggregated (one atomic per warp per archetype);
//   * entity IDs come from per-world caches that replay the CPU backend's
//     IDMap algorithm (include/madrona/impl/id_map_impl.inl:69-225), so IDs
//     match the CPU oracle bit-for-bit instead of being atomic-order dependent.
#pragma once

#include <cstdint>
#include <new>
#include <madrona/ecs.hpp>
#include <madrona/ecs_flags.hpp>
#include <madrona/type_tracker.hpp>
#include <madrona/optional.hpp>
#include <madrona/span.hpp>
#include <mb2_state.h>

namespace madrona {

namespace mwGPU {

template <int... Is> struct IntList {};
template <int N, int... Is> struct MakeIntList : MakeIntList<N - 1, N - 1, Is...> {};
template <int... Is> struct MakeIntList<0, Is...> { using type = IntList<Is...>; };
template <int N> using IntSeq = typename MakeIntList<N>::type;

// Set by the host right after the module is loaded.
extern "C" __constant__ mb2::EngineState *mb2_engine_state;

inline mb2::EngineState &engine() { return *mb2_engine_state; }

inline void raiseError(uint32_t flag, uint32_t archetype = 0)
{
    mb2::EngineState &S = engine();
    atomicOr(&S.errorFlags, flag);
    S.errorArchetype = archetype;
}

// ---- per-world entity ID cache (IDMap::Cache replay) ----------------------

inline void lockCache(mb2::IDCache &c)
{
    while (atomicCAS(&c.lock, 0, 1) != 0) {}
    __threadfence();
}

inline void unlockCache(mb2::IDCache &c)
{
    __threadfence();
    atomicExch(&c.lock, 0);
}

// Pop the head of a cached sub-list; FreeNode.globalNext (= slot.b) doubles
// as a run length of contiguous never-used IDs (id_map_impl.inl:72-101).
inline Entity popCachedID(mb2::EntitySlot *slots, int32_t *head)
{
    int32_t id = *head;
    mb2::EntitySlot node = slots[id];
    if (node.b == 1) {
        *head = node.a;
    } else {
        int32_t next = id + 1;
        slots[next].a = node.a;
        slots[next].b = node.b - 1;
        slots[next].gen = 0;
        *head = next;
    }
    return Entity { node.gen, id };
}

inline Entity acquireEntityLocked(mb2::EngineState &S, mb2::IDCache &c)
{
    mb2::EntitySlot *slots = S.entitySlots;

    if (c.numOverflow > 0) {
        c.numOverflow -= 1;
        return popCachedID(slots, &c.overflowHead);
    }
    if (c.numFree > 0) {
        c.numFree -= 1;
        return popCachedID(slots, &c.freeHead);
    }

    // Refill from the global free list: 64-bit {gen, head} CAS.
    unsigned long long *head_ptr = (unsigned long long *)&S.freeHead;
    unsigned long long cur = *(volatile unsigned long long *)head_ptr;
    int32_t got = mb2::kIDSentinel;
    while (true) {
        int32_t head = (int32_t)(uint32_t)(cur & 0xFFFFFFFFull);
        if (head == mb2::kIDSentinel) break;
        uint32_t gen = (uint32_t)(cur >> 32);
        int32_t next = ((volatile mb2::EntitySlot *)slots)[head].b;
        unsigned long long want =
            ((unsigned long long)(gen + 1) << 32) | (uint32_t)next;
        unsigned long long prev = atomicCAS(head_ptr, cur, want);
        if (prev == cur) { got = head; break; }
        cur = prev;
    }

    if (got != mb2::kIDSentinel) {
        slots[got].b = 1;
        c.freeHead = got;
        c.numFree = mb2::kIDsPerCache - 1;
        return popCachedID(slots, &c.freeHead);
    }

    // Expand the store by one 64-ID block.  During the second init pass the
    // block index is pre-assigned in world order so that IDs equal those of
    // the reference's sequential per-world construction (mw_cpu.inl:40-44).
    int32_t block_start;
    if (S.initPass == 1) {
        block_start = (c.expandBase + c.numExpands) * mb2::kIDsPerCache;
    } else {
        block_start = atomicAdd(&S.numEntitySlots, mb2::kIDsPerCache);
    }
    c.numExpands += 1;

    if (block_start + mb2::kIDsPerCache > S.entityCapacity) {
        raiseError(mb2::ErrEntityOverflow);
        return Entity::none();
    }

    slots[block_start].gen = 0;
    int32_t free_start = block_start + 1;
    slots[free_start].a = mb2::kIDSentinel;
    slots[free_start].b = mb2::kIDsPerCache - 1;
    slots[free_start].gen = 0;
    c.freeHead = free_start;
    c.numFree = mb2::kIDsPerCache - 1;
    return Entity { 0, block_start };
}

inline void releaseEntityLocked(mb2::EngineState &S, mb2::IDCache &c, int32_t id)
{
    mb2::EntitySlot *slots = S.entitySlots;
    slots[id].gen += 1;
    slots[id].b = 1;

    if (c.numFree < mb2::kIDsPerCache) {
        slots[id].a = c.freeHead;
        c.freeHead = id;
        c.numFree += 1;
        return;
    }
    if (c.numOverflow < mb2::kIDsPerCache) {
        slots[id].a = c.overflowHead;
        c.overflowHead = id;
        c.numOverflow += 1;
    }
    if (c.numOverflow == mb2::kIDsPerCache) {
        unsigned long long *head_ptr = (unsigned long long *)&S.freeHead;
        unsigned long long cur = *(volatile unsigned long long *)head_ptr;
        while (true) {
            uint32_t gen = (uint32_t)(cur >> 32);
            slots[c.overflowHead].b = (int32_t)(uint32_t)(cur & 0xFFFFFFFFull);
            __threadfence();
            unsigned long long want =
                ((unsigned long long)(gen + 1) << 32) | (uint32_t)c.overflowHead;
            unsigned long long prev = atomicCAS(head_ptr, cur, want);
            if (prev == cur) break;
            cur = prev;
        }
        c.overflowHead = mb2::kIDSentinel;
        c.numOverflow = 0;
    }
}

// Warp-aggregated row append: lanes of the warp that append to the same
// archetype at the same time share one atomicAdd; rows are handed out in lane
// order (so, for one-thread-per-world systems, in world order).
inline int32_t appendRow(mb2::TableDesc &tbl, uint32_t archetype_id)
{
    unsigned active = __activemask();
    unsigned peers = __match_any_sync(active, archetype_id);
    unsigned lane = threadIdx.x & 31u;
    int leader = __ffs(peers) - 1;
    int rank = __popc(peers & ((1u << lane) - 1u));
    int32_t base = 0;
    if ((int)lane == leader) {
        const int32_t count = __popc(peers);
        base = atomicAdd(&tbl.numRows, count);
        tbl.needsSort = 1;
        // overflow: pull the row count back to the capacity so the later nodes
        // of the same graph (which size their loops and scratch by numRows)
        // stay inside the allocation; the step still reports the error
        if (base + count > tbl.capacity) atomicMin(&tbl.numRows, tbl.capacity);
    }
    base = __shfl_sync(peers, base, leader);
    int32_t row = base + rank;
    if (row >= tbl.capacity) {
        // The step is reported as failed (run() returns the error); the caller
        // still gets a row INSIDE the allocation -- the table's last one, shared
        // by every overflowing append -- so simulator code that goes on to
        // initialise "its" new entity cannot write out of bounds.
        raiseError(mb2::ErrTableOverflow, archetype_id);
        return tbl.capacity - 1;
    }
    return row;
}

inline Loc lookupLoc(mb2::EngineState &S, Entity e)
{
    if (e.id < 0 || e.id >= S.entityCapacity) return Loc::none();
    mb2::EntitySlot s = S.entitySlots[e.id];
    if (s.gen != e.gen) return Loc::none();
    return Loc { (uint32_t)s.a, s.b };
}

}

template <typename T>
class ResultRef {
public:
    inline ResultRef(T *ptr) : ptr_(ptr) {}
    inline bool valid() const { return ptr_ != nullptr; }
    inline T &value() { return *ptr_; }
private:
    T *ptr_;
};

template <typename SingletonT>
struct SingletonArchetype : public Archetype<SingletonT> {};

// Per-instantiation query cache: [archetype, col...] tuples, ascending
// archetype ID (reference: src/core/state.cpp:271-363).  QueryRef is the
// component-count-independent head that custom nodes keep a pointer to
// (Query::getSharedRef, reference: include/madrona/query.hpp:17-43).
struct QueryRef {
    static constexpr int maxArchetypes = 12;
    int32_t resolved;
    int32_t numArchetypes;
    int32_t numComponents;
    int32_t archetypes[maxArchetypes];
};

template <int N>
struct QueryData : QueryRef {
    int32_t cols[maxArchetypes][N];
};

template <typename... ComponentTs>
__device__ QueryData<(int)sizeof...(ComponentTs)> mb2QueryStorage = {};

template <typename... ComponentTs>
class Query {
public:
    static inline QueryData<(int)sizeof...(ComponentTs)> &data()
    {
        return mb2QueryStorage<ComponentTs...>;
    }
    inline Query() {}
    inline uint32_t numMatchingArchetypes() const { return (uint32_t)data().numArchetypes; }
    inline QueryRef *getSharedRef() const { return &data(); }
};

// The subset of the reference StateManager surface that library/simulator
// code reaches through mwGPU::getStateManager() (state.hpp:122-170).
class StateManager {
public:
    template <typename ComponentT>
    inline ComponentID registerComponent(uint32_t num_bytes = 0);

    template <typename ArchetypeT, typename... MetadataComponentTs>
    inline ArchetypeID registerArchetype(
        ComponentMetadataSelector<MetadataComponentTs...> component_metadatas,
        ArchetypeFlags archetype_flags, CountT max_num_entities_per_world);

    template <typename BundleT> inline void registerBundle();
    template <typename AliasT, typename BundleT> inline void registerBundleAlias();
    template <typename SingletonT> inline void registerSingleton();

    template <typename ComponentT>
    inline ComponentID componentID() const { return { TypeTracker::typeID<ComponentT>() }; }
    template <typename ArchetypeT>
    inline ArchetypeID archetypeID() const { return { TypeTracker::typeID<ArchetypeT>() }; }

    inline Loc getLoc(Entity e) const { return mwGPU::lookupLoc(mwGPU::engine(), e); }

    inline int32_t columnIndex(uint32_t archetype_id, uint32_t component_id) const
    {
        return mwGPU::engine().columnLookup[archetype_id][component_id];
    }

    template <typename ComponentT>
    inline ComponentT *getArchetypeComponent(uint32_t archetype_id)
    {
        mb2::EngineState &S = mwGPU::engine();
        int32_t col = S.columnLookup[archetype_id][TypeTracker::typeID<ComponentT>()];
        return (ComponentT *)S.tables[archetype_id].columns[col];
    }

    template <typename ArchetypeT, typename ComponentT>
    inline ComponentT *getArchetypeComponent()
    {
        return getArchetypeComponent<ComponentT>(TypeTracker::typeID<ArchetypeT>());
    }

    inline void *getArchetypeColumn(uint32_t archetype_id, int32_t col)
    {
        return mwGPU::engine().tables[archetype_id].columns[col];
    }

    template <typename ArchetypeT>
    inline int32_t *getArchetypeWorldOffsets()
    {
        return mwGPU::engine().tables[TypeTracker::typeID<ArchetypeT>()].worldOffsets;
    }
    template <typename ArchetypeT>
    inline int32_t *getArchetypeWorldCounts()
    {
        return mwGPU::engine().tables[TypeTracker::typeID<ArchetypeT>()].worldCounts;
    }
    template <typename ArchetypeT>
    inline int32_t getArchetypeNumRows()
    {
        return mwGPU::engine().tables[TypeTracker::typeID<ArchetypeT>()].numRows;
    }

    template <typename ArchetypeT, typename ComponentT>
    inline ComponentT *getWorldComponents(uint32_t world_id)
    {
        mb2::TableDesc &t = mwGPU::engine().tables[TypeTracker::typeID<ArchetypeT>()];
        return getArchetypeComponent<ArchetypeT, ComponentT>() + t.worldOffsets[world_id];
    }
    template <typename ArchetypeT>
    inline Entity *getWorldEntities(uint32_t world_id)
    {
        mb2::TableDesc &t = mwGPU::engine().tables[TypeTracker::typeID<ArchetypeT>()];
        return (Entity *)t.columns[0] + t.worldOffsets[world_id];
    }
    template <typename ArchetypeT>
    inline CountT numRows(uint32_t world_id)
    {
        return mwGPU::engine().tables[TypeTracker::typeID<ArchetypeT>()].worldCounts[world_id];
    }

    inline uint32_t numWorlds() const { return mwGPU::engine().numWorlds; }

    template <typename... ComponentTs>
    inline void resolveQuery(QueryData<(int)sizeof...(ComponentTs)> &q);

    // ---- read side for custom nodes (reference: src/mw/device/include/madrona/state.hpp
    // :83-181, state.inl:160-272).  Row counts include rows destroyed since the table's
    // last sort or compaction (their WorldID is -1), as in the reference.
    template <typename... ComponentTs>
    inline Query<ComponentTs...> query()
    {
        auto &q = Query<ComponentTs...>::data();
        if (((volatile int32_t *)&q.resolved)[0] == 0) resolveQuery<ComponentTs...>(q);
        return Query<ComponentTs...>();
    }

    // fn(numRows, WorldID *worldColumn, void *column...) per matching archetype; a true
    // return stops the iteration
    template <int32_t num_components, typename Fn>
    inline void iterateArchetypesRaw(QueryRef *query_ref, Fn &&fn)
    {
        iterateArchetypesRawImpl<num_components>(query_ref, fn, mwGPU::IntSeq<num_components> {});
    }

    inline uint32_t numMatchingEntities(QueryRef *query_ref)
    {
        mb2::EngineState &S = mwGPU::engine();
        uint32_t total = 0;
        for (int32_t i = 0; i < query_ref->numArchetypes; i++) {
            total += (uint32_t)S.tables[query_ref->archetypes[i]].numRows;
        }
        return total;
    }

    inline void *getArchetypeComponent(uint32_t archetype_id, uint32_t component_id)
    {
        return getArchetypeColumn(archetype_id, getArchetypeColumnIndex(archetype_id, component_id));
    }
    inline int32_t getArchetypeColumnIndex(uint32_t archetype_id, uint32_t component_id)
    {
        return mwGPU::engine().columnLookup[archetype_id][component_id];
    }
    inline uint32_t getArchetypeColumnBytesPerRow(uint32_t archetype_id, int32_t column_idx)
    {
        return mwGPU::engine().tables[archetype_id].columnBytes[column_idx];
    }
    inline int32_t getArchetypeNumColumns(uint32_t archetype_id)
    {
        return mwGPU::engine().tables[archetype_id].numColumns;
    }
    inline int32_t *getArchetypeWorldOffsets(uint32_t archetype_id)
    {
        return mwGPU::engine().tables[archetype_id].worldOffsets;
    }
    inline int32_t *getArchetypeWorldCounts(uint32_t archetype_id)
    {
        return mwGPU::engine().tables[archetype_id].worldCounts;
    }
    inline int32_t numArchetypeRows(uint32_t archetype_id) const
    {
        return mwGPU::engine().tables[archetype_id].numRows;
    }

private:
    template <int32_t num_components, typename Fn, int... Is>
    inline void iterateArchetypesRawImpl(QueryRef *query_ref, Fn &fn, mwGPU::IntList<Is...>)
    {
        mb2::EngineState &S = mwGPU::engine();
        auto *q = static_cast<QueryData<num_components> *>(query_ref);
        for (int32_t i = 0; i < q->numArchetypes; i++) {
            mb2::TableDesc &t = S.tables[q->archetypes[i]];
            if (fn(t.numRows, (WorldID *)t.columns[1], t.columns[q->cols[i][Is]]...)) return;
        }
    }
};

namespace mwGPU {
inline StateManager *getStateManager()
{
    // Stateless facade: all state lives in mb2::EngineState.
    return (StateManager *)(void *)mb2_engine_state;
}
}

// ---- registration (runs on the device in a 1-thread kernel) ----------------

template <typename ComponentT>
ComponentID StateManager::registerComponent(uint32_t num_bytes)
{
    mb2::EngineState &S = mwGPU::engine();
    TypeTracker::registerType<ComponentT>(&S.numComponents);
    uint32_t id = TypeTracker::typeID<ComponentT>();
    if (id >= (uint32_t)mb2::kMaxComponents) {
        mwGPU::raiseError(mb2::ErrRegistry);
        return { id };
    }
    uint32_t bytes = num_bytes == 0 ? (uint32_t)sizeof(ComponentT) : num_bytes;
    S.components[id].numBytes = bytes;
    S.components[id].alignment = (uint32_t)alignof(ComponentT);
    return { id };
}

namespace mwGPU {
template <typename T> struct PackIDs;
template <template <typename...> class P, typename... Ts>
struct PackIDs<P<Ts...>> {
    static constexpr int count = (int)sizeof...(Ts);
    static inline void fill(uint32_t *out)
    {
        uint32_t ids[sizeof...(Ts) == 0 ? 1 : sizeof...(Ts)] = { TypeTracker::typeID<Ts>()... };
        for (int i = 0; i < count; i++) out[i] = ids[i];
    }
};
}

template <typename ArchetypeT, typename... MetadataComponentTs>
ArchetypeID StateManager::registerArchetype(
    ComponentMetadataSelector<MetadataComponentTs...>,
    ArchetypeFlags archetype_flags, CountT max_num_entities_per_world)
{
    mb2::EngineState &S = mwGPU::engine();
    TypeTracker::registerType<ArchetypeT>(&S.numArchetypes);
    uint32_t id = TypeTracker::typeID<ArchetypeT>();
    if (id >= (uint32_t)mb2::kMaxArchetypes) {
        mwGPU::raiseError(mb2::ErrRegistry);
        return { id };
    }

    using Pack = mwGPU::PackIDs<typename ArchetypeT::Base>;
    uint32_t listed[Pack::count == 0 ? 1 : Pack::count];
    Pack::fill(listed);

    mb2::ArchetypeInfo &info = S.archetypes[id];
    uint32_t n = 0;
    for (int i = 0; i < Pack::count; i++) {
        uint32_t cid = listed[i];
        if (cid == TypeTracker::unassignedTypeID) {
            mwGPU::raiseError(mb2::ErrRegistry, id);
            continue;
        }
        if (cid & mb2::kBundleMask) {
            // bundles are flattened in place (src/core/state.cpp:408-426)
            const mb2::BundleInfo &b = S.bundles[cid & ~mb2::kBundleMask];
            for (uint32_t j = 0; j < b.numComponents; j++) {
                if (n < (uint32_t)mb2::kMaxColumns - 2) info.componentIDs[n++] = b.componentIDs[j];
            }
        } else if (n < (uint32_t)mb2::kMaxColumns - 2) {
            info.componentIDs[n++] = cid;
        }
    }
    info.numUserComponents = n;
    info.flags = (uint32_t)archetype_flags;
    info.maxPerWorld = (int32_t)max_num_entities_per_world;
    info.isSingleton = 0;
    info.registered = 1;
    return { id };
}

template <typename BundleT>
void StateManager::registerBundle()
{
    mb2::EngineState &S = mwGPU::engine();
    if (TypeTracker::typeID<BundleT>() != TypeTracker::unassignedTypeID) return;

    uint32_t next = S.numBundles | mb2::kBundleMask;
    TypeTracker::registerType<BundleT>(&next);
    S.numBundles = next & ~mb2::kBundleMask;
    uint32_t id = TypeTracker::typeID<BundleT>() & ~mb2::kBundleMask;
    if (id >= (uint32_t)mb2::kMaxBundles) {
        mwGPU::raiseError(mb2::ErrRegistry);
        return;
    }

    using Pack = mwGPU::PackIDs<typename BundleT::Base>;
    uint32_t listed[Pack::count == 0 ? 1 : Pack::count];
    Pack::fill(listed);

    mb2::BundleInfo &b = S.bundles[id];
    uint32_t n = 0;
    for (int i = 0; i < Pack::count; i++) {
        uint32_t cid = listed[i];
        if (cid & mb2::kBundleMask) {
            const mb2::BundleInfo &sub = S.bundles[cid & ~mb2::kBundleMask];
            for (uint32_t j = 0; j < sub.numComponents; j++) {
                if (n < (uint32_t)mb2::kMaxBundleComponents) b.componentIDs[n++] = sub.componentIDs[j];
            }
        } else if (n < (uint32_t)mb2::kMaxBundleComponents) {
            b.componentIDs[n++] = cid;
        }
    }
    b.numComponents = n;
    b.registered = 1;
}

template <typename AliasT, typename BundleT>
void StateManager::registerBundleAlias()
{
    if (TypeTracker::typeID<AliasT>() != TypeTracker::unassignedTypeID) return;
    uint32_t bundle_id = TypeTracker::typeID<BundleT>();
    TypeTracker::registerType<AliasT>(&bundle_id);
}

template <typename SingletonT>
void StateManager::registerSingleton()
{
    using ArchetypeT = SingletonArchetype<SingletonT>;
    registerComponent<SingletonT>();
    ArchetypeID id = registerArchetype<ArchetypeT>(
        ComponentMetadataSelector<> {}, ArchetypeFlags::None, 1);
    mb2::EngineState &S = mwGPU::engine();
    S.archetypes[id.id].isSingleton = 1;
    S.archetypes[id.id].singletonOrder = S.numSingletons++;
}

template <typename... ComponentTs>
void StateManager::resolveQuery(QueryData<(int)sizeof...(ComponentTs)> &q)
{
    constexpr int N = (int)sizeof...(ComponentTs);
    mb2::EngineState &S = mwGPU::engine();
    uint32_t ids[N] = { TypeTracker::typeID<ComponentTs>()... };
    int found = 0;
    for (uint32_t a = 0; a < S.numArchetypes; a++) {
        if (!S.archetypes[a].registered) continue;
        int32_t cols[N];
        bool ok = true;
        for (int i = 0; i < N; i++) {
            int32_t c = ids[i] < (uint32_t)mb2::kMaxComponents ?
                S.columnLookup[a][ids[i]] : -1;
            if (c < 0) { ok = false; break; }
            cols[i] = c;
        }
        if (!ok) continue;
        if (found < QueryData<N>::maxArchetypes) {
            q.archetypes[found] = (int32_t)a;
            for (int i = 0; i < N; i++) q.cols[found][i] = cols[i];
            found++;
        }
    }
    q.numArchetypes = found;
    q.numComponents = N;
    __threadfence();
    q.resolved = 1;
}

}
