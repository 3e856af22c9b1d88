// TaskGraph construction API (reference: include/madrona/taskgraph_builder.hpp
// :22-219; GPU node set src/mw/device/include/madrona/taskgraph.hpp:207-381).
//
// There is no megakernel here.  setupTasks runs once on the device (1 thread)
// and appends mb2::NodeRecords; every ParallelForNode instantiation owns a
// real __global__ kernel (mwGPU::nodeKern<NodeT>) that the host launches as a
// CUDA-graph kernel node.  The host pairs records with kernels through the
// address of mwGPU::nodeMeta<NodeT>, whose mangled name shares the <NodeT>
// encoding with the kernel's.
//
// Custom node types (reference GPU API: src/mw/device/include/madrona/taskgraph.hpp
// :28-132, taskgraph.inl:43-162) work the same way: addNodeFn<fn> records a
// NodeUserFn whose kernel is nodeKern<FnNode<NodeT, fn>>.  Node data lives in
// 256-byte device slots (EngineState::nodeData) that setupTasks constructs in
// place, so TaskGraphBuilder::getDataRef and TaskGraph::getNodeData name the
// same memory.
#pragma once
#include <utility>
#include <madrona/fwd.hpp>
#include <madrona/context.hpp>
#include <madrona/custom_context.hpp>

namespace madrona {

struct NodeBase {
    // Invocations of the next run of a node added with a fixed count of 0.  It is read
    // once, after the node's dependencies finished and before any invocation runs.
    uint32_t numDynamicInvocations;
};

struct TaskGraphNodeID {
    uint32_t id;
};

class TaskGraphBuilder;

namespace mwGPU {

inline char *nodeDataSlot(int32_t data_idx)
{
    return engine().nodeData + (size_t)data_idx * mb2::kNodeDataBytes;
}

template <typename C, typename D>
D *contextDataPtr(CustomContext<C, D> *);
WorldBase *contextDataPtr(Context *);

}

// Run-time side of custom nodes.  Every task graph shares the node data array, so
// this is a stateless facade (like StateManager) that mwGPU::getTaskGraph returns.
class TaskGraph {
public:
    static inline constexpr uint32_t maxNodeDataBytes = mb2::kNodeDataBytes;

    using NodeID = TaskGraphNodeID;
    using Builder = TaskGraphBuilder;

    struct DataID {
        int32_t id;
    };

    template <typename NodeT>
    struct TypedDataID : DataID {};

    static inline WorldBase *getWorld(int32_t world_idx)
    {
        mb2::EngineState &S = mwGPU::engine();
        return (WorldBase *)(S.worldData + (size_t)world_idx * S.worldDataStride);
    }

    template <typename ContextT>
    static inline ContextT makeContext(WorldID world_id)
    {
        using DataT = decltype(mwGPU::contextDataPtr((ContextT *)nullptr));
        return ContextT((DataT)getWorld(world_id.idx), WorkerInit { world_id });
    }

    template <typename NodeT>
    inline NodeT &getNodeData(TypedDataID<NodeT> data_id)
    {
        return *(NodeT *)mwGPU::nodeDataSlot(data_id.id);
    }
};

namespace mwGPU {

inline TaskGraph &getTaskGraph(uint32_t)
{
    return *(TaskGraph *)(void *)mb2_engine_state;
}

template <typename NodeT>
__device__ uint32_t nodeMeta = 0;

template <typename NodeT>
__global__ void __launch_bounds__(256) nodeKern(const mb2::NodeRecord *rec)
{
    NodeT::run(*rec);
}

template <auto K> struct KernelInstantiate { static constexpr int v = 1; };

template <typename T> struct RemovePtr { using type = T; };
template <typename T> struct RemovePtr<T *> { using type = T; };

// std::invoke(fn, node, invocation) without <functional> (reference: userEntry,
// taskgraph.inl:12-19): member functions of the node type and free functions
// taking (NodeT *, int32_t)
template <typename NodeT, typename R, typename C, typename A>
inline void invokeNodeFn(R (C::*fn)(A), NodeT *node, int32_t invocation) { (node->*fn)(invocation); }
template <typename NodeT, typename R, typename C, typename A>
inline void invokeNodeFn(R (C::*fn)(A) const, NodeT *node, int32_t invocation) { (node->*fn)(invocation); }
template <typename NodeT, typename Fn>
inline void invokeNodeFn(Fn fn, NodeT *node, int32_t invocation) { fn(node, invocation); }

// Tag type of a custom node's kernel, nodeKern<FnNode<NodeT, fn>>.  The host launches
// 256-thread blocks; invocation i runs on threads i*tpi .. i*tpi+tpi-1 of a grid-stride
// loop.  tpi divides 256, so an invocation never straddles a block: with tpi = 256 the
// loop is block-uniform (__shared__ and __syncthreads() are fine), with tpi = 32 warp-uniform.
template <typename NodeT, auto fn>
struct FnNode {
    static inline void run(const mb2::NodeRecord &rec)
    {
        NodeT *node = (NodeT *)nodeDataSlot((int32_t)rec.userFn.dataIdx);
        const uint32_t tpi = rec.userFn.threadsPerInvocation;
        const uint64_t n = rec.userFn.fixedCount != 0 ? rec.userFn.fixedCount : rec.userFn.latchedCount;
        const uint64_t stride = (gridDim.x * blockDim.x) / tpi;
        for (uint64_t inv = (blockIdx.x * blockDim.x + threadIdx.x) / tpi; inv < n; inv += stride) {
            invokeNodeFn<NodeT>(fn, node, (int32_t)inv);
        }
    }
};

}

class TaskGraphBuilder {
public:
    inline TaskGraphBuilder() : taskgraph_id_(0) {}

    template <typename NodeT>
    inline TaskGraphNodeID addToGraph(Span<const TaskGraphNodeID> dependencies)
    {
        return NodeT::addToGraph(*this, dependencies);
    }

    // Append a record; returns its (global) node index.
    inline TaskGraphNodeID pushNode(const mb2::NodeRecord &proto,
                                    Span<const TaskGraphNodeID> dependencies)
    {
        mb2::EngineState &S = mwGPU::engine();
        if (S.numNodes >= (uint32_t)mb2::kMaxNodes) {
            mwGPU::raiseError(mb2::ErrTooManyNodes);
            return { S.numNodes - 1 };
        }
        uint32_t idx = S.numNodes++;
        mb2::NodeRecord &r = S.nodes[idx];
        r = proto;
        r.taskgraph = taskgraph_id_;
        r.numDeps = 0;
        for (CountT i = 0; i < dependencies.size() && i < mb2::kMaxNodeDeps; i++) {
            r.deps[r.numDeps++] = dependencies[i].id;
        }
        return { idx };
    }

    inline uint32_t taskgraphID() const { return taskgraph_id_; }
    inline uint32_t getTaskgraphID() const { return taskgraph_id_; }

    // ---- custom nodes (reference: src/mw/device/include/madrona/taskgraph.inl:43-124)
    using DataID = TaskGraph::DataID;
    template <typename NodeT>
    using TypedDataID = TaskGraph::TypedDataID<NodeT>;

    // A zero-filled 256-byte slot with NodeT constructed in it.  Past kMaxNodeDatas the
    // executor fails to build; until then the extra constructs share one spare slot.
    template <typename NodeT, typename... Args>
    inline TypedDataID<NodeT> constructNodeData(Args &&...args)
    {
        static_assert(sizeof(NodeT) <= TaskGraph::maxNodeDataBytes);
        static_assert(alignof(NodeT) <= TaskGraph::maxNodeDataBytes);
        mb2::EngineState &S = mwGPU::engine();
        int32_t idx = (int32_t)S.numNodeDatas;
        if (idx >= mb2::kMaxNodeDatas) {
            mwGPU::raiseError(mb2::ErrTooManyNodeDatas);
            idx = mb2::kMaxNodeDatas;
        } else {
            S.numNodeDatas++;
        }
        char *slot = mwGPU::nodeDataSlot(idx);
        for (int i = 0; i < mb2::kNodeDataBytes / 8; i++) ((uint64_t *)slot)[i] = 0;
        new (slot) NodeT(std::forward<Args>(args)...);
        return TypedDataID<NodeT> { DataID { idx } };
    }

    template <typename NodeT>
    inline NodeT &getDataRef(TypedDataID<NodeT> data_id)
    {
        return *(NodeT *)mwGPU::nodeDataSlot(data_id.id);
    }

    // fn(NodeT *, int32_t invocation) runs fixed_num_invocations times, or, with 0, as many
    // times as the data's numDynamicInvocations says when the node starts.  The data must
    // begin with its NodeBase (no virtual functions), where the engine latches the count.
    // num_threads_per_invocation must divide 256.  parent_node only orders, as one more
    // dependency (the reference merely counts children with it).
    template <auto fn, typename NodeT>
    inline TaskGraphNodeID addNodeFn(TypedDataID<NodeT> data,
                                     Span<const TaskGraphNodeID> dependencies,
                                     Optional<TaskGraphNodeID> parent_node =
                                         Optional<TaskGraphNodeID>::none(),
                                     uint32_t fixed_num_invocations = 0,
                                     uint32_t num_threads_per_invocation = 1)
    {
        using Tag = mwGPU::FnNode<NodeT, fn>;
        static_assert(mwGPU::KernelInstantiate<&mwGPU::nodeKern<Tag>>::v == 1);
        static_assert(!__is_polymorphic(NodeT));

        mb2::NodeRecord rec {};
        rec.kind = mb2::NodeUserFn;
        rec.userFn.dataIdx = (uint32_t)data.id;
        rec.userFn.fixedCount = fixed_num_invocations;
        rec.userFn.threadsPerInvocation = num_threads_per_invocation;
        unsigned long long meta_addr = (unsigned long long)(void *)&mwGPU::nodeMeta<Tag>;
        rec.kernelID = (uint32_t)(meta_addr & 0xFFFFFFFFull);
        rec.component = (uint32_t)(meta_addr >> 32);

        TaskGraphNodeID deps[mb2::kMaxNodeDeps];
        CountT n = 0;
        for (CountT i = 0; i < dependencies.size() && n < mb2::kMaxNodeDeps; i++) deps[n++] = dependencies[i];
        if (parent_node.has_value() && n < mb2::kMaxNodeDeps) deps[n++] = *parent_node;
        return pushNode(rec, Span<const TaskGraphNodeID>(deps, n));
    }

    template <typename NodeT, int32_t count = 1, typename... Args>
    inline TaskGraphNodeID addOneOffNode(Span<const TaskGraphNodeID> dependencies, Args &&...args)
    {
        auto data_id = constructNodeData<NodeT>(std::forward<Args>(args)...);
        return addNodeFn<&NodeT::run>(data_id, dependencies, Optional<TaskGraphNodeID>::none(),
                                      (uint32_t)count);
    }

    // A one-invocation node sets numDynamicInvocations = numInvocations(); NodeT::run
    // follows it with a dynamic count.
    template <typename NodeT, typename... Args>
    inline TaskGraphNodeID addDynamicCountNode(Span<const TaskGraphNodeID> dependencies,
                                               uint32_t num_threads_per_invocation, Args &&...args)
    {
        auto data_id = constructNodeData<NodeT>(std::forward<Args>(args)...);
        TaskGraphNodeID count_node = addNodeFn<&TaskGraphBuilder::dynamicCountWrapper<NodeT>>(
            data_id, dependencies, Optional<TaskGraphNodeID>::none(), 1);
        return addNodeFn<&NodeT::run>(data_id, { count_node }, Optional<TaskGraphNodeID>::none(), 0,
                                      num_threads_per_invocation);
    }

private:
    template <typename NodeT>
    static inline void dynamicCountWrapper(NodeT *node, int32_t)
    {
        node->numDynamicInvocations = (uint32_t)node->numInvocations();
    }

    uint32_t taskgraph_id_;
friend class TaskGraphManager;
};

class TaskGraphManager {
public:
    inline TaskGraphManager(uint32_t num_taskgraphs) : num_(num_taskgraphs) {}

    template <EnumType EnumT>
    inline TaskGraphBuilder &init(EnumT taskgraph_id) { return init((uint32_t)taskgraph_id); }

    inline TaskGraphBuilder &init(uint32_t taskgraph_id)
    {
        builders_[taskgraph_id].taskgraph_id_ = taskgraph_id;
        return builders_[taskgraph_id];
    }

private:
    TaskGraphBuilder builders_[mb2::kMaxTaskGraphs];
    uint32_t num_;
};

// ---- ParallelFor ----------------------------------------------------------
// One record (and one launch) per archetype matching the component list; the
// kernel grid-strides over the table's live row count read on the device, so
// the captured CUDA graph never needs a host-side size.
template <typename ContextT, auto Fn, int threads_per_invocation,
          int items_per_invocation, typename... ComponentTs>
class CustomParallelForNode : public NodeBase {
public:
    static inline void run(const mb2::NodeRecord &rec)
    {
        runImpl(rec, mwGPU::IntSeq<(int)sizeof...(ComponentTs)> {});
    }

    static inline TaskGraphNodeID addToGraph(
        TaskGraphBuilder &builder, Span<const TaskGraphNodeID> dependencies)
    {
        using Self = CustomParallelForNode;
        static_assert(mwGPU::KernelInstantiate<&mwGPU::nodeKern<Self>>::v == 1);
        static_assert(sizeof...(ComponentTs) <= (size_t)mb2::kMaxNodeCols);

        auto &q = Query<ComponentTs...>::data();
        if (q.resolved == 0) {
            mwGPU::getStateManager()->template resolveQuery<ComponentTs...>(q);
        }

        mb2::NodeRecord rec {};
        rec.kind = mb2::NodeUserParallelFor;
        rec.numCols = (int32_t)sizeof...(ComponentTs);
        rec.userTag = (uint32_t)threads_per_invocation;
        // identity of this instantiation for the host (see header comment)
        unsigned long long meta_addr =
            (unsigned long long)(void *)&mwGPU::nodeMeta<Self>;
        rec.kernelID = (uint32_t)(meta_addr & 0xFFFFFFFFull);
        rec.component = (uint32_t)(meta_addr >> 32);

        TaskGraphNodeID last { 0xFFFFFFFFu };
        Span<const TaskGraphNodeID> deps = dependencies;
        for (int qa = 0; qa < q.numArchetypes; qa++) {
            rec.archetype = (uint32_t)q.archetypes[qa];
            for (int i = 0; i < rec.numCols; i++) rec.cols[i] = q.cols[qa][i];
            last = builder.pushNode(rec, deps);
        }
        if (q.numArchetypes == 0) {
            // nothing matches: keep a no-op record so dependency IDs stay valid
            rec.kind = mb2::NodeResetTmpAlloc;
            rec.userTag = 0xFFFFFFFFu;
            last = builder.pushNode(rec, deps);
        }
        return last;
    }

private:
    template <int... Is>
    static inline void runImpl(const mb2::NodeRecord &rec, mwGPU::IntList<Is...>)
    {
        using DataT = typename mwGPU::RemovePtr<
            decltype(mwGPU::contextDataPtr((ContextT *)nullptr))>::type;
        mb2::EngineState &S = mwGPU::engine();
        const mb2::TableDesc &t = S.tables[rec.archetype];
        const int32_t n = t.numRows;
        const WorldID *world_col = (const WorldID *)t.columns[1];
        const int32_t stride =
            (int32_t)((gridDim.x * blockDim.x) / threads_per_invocation);
        int32_t row =
            (int32_t)((blockIdx.x * blockDim.x + threadIdx.x) / threads_per_invocation);
        for (; row < n; row += stride) {
            WorldID w = world_col[row];
            if (w.idx < 0) continue;   // destroyed row awaiting compaction
            ContextT ctx((DataT *)(S.worldData + (size_t)w.idx * S.worldDataStride),
                         WorkerInit { w });
            Fn(ctx, ((ComponentTs *)t.columns[rec.cols[Is]])[row]...);
        }
    }
};

template <typename ContextT, auto Fn, typename... ComponentTs>
using ParallelForNode = CustomParallelForNode<ContextT, Fn, 1, 1, ComponentTs...>;

// ---- engine-owned nodes: recorded here, executed by ahead-of-time kernels --
namespace mwGPU {
inline TaskGraphNodeID pushBuiltin(TaskGraphBuilder &builder,
                                   Span<const TaskGraphNodeID> deps,
                                   uint32_t kind, uint32_t archetype = 0,
                                   uint32_t component = 0, uint32_t tag = 0)
{
    mb2::NodeRecord rec {};
    rec.kind = kind;
    rec.archetype = archetype;
    rec.component = component;
    rec.userTag = tag;
    return builder.pushNode(rec, deps);
}
}

class ResetTmpAllocNode : public NodeBase {
public:
    static inline TaskGraphNodeID addToGraph(
        TaskGraphBuilder &builder, Span<const TaskGraphNodeID> deps)
    {
        return mwGPU::pushBuiltin(builder, deps, mb2::NodeResetTmpAlloc);
    }
};

template <typename ArchetypeT>
class ClearTmpNode : public NodeBase {
public:
    static inline TaskGraphNodeID addToGraph(
        TaskGraphBuilder &builder, Span<const TaskGraphNodeID> deps)
    {
        return mwGPU::pushBuiltin(builder, deps, mb2::NodeClearTmp,
                                  TypeTracker::typeID<ArchetypeT>());
    }
};

class RecycleEntitiesNode : public NodeBase {
public:
    static inline TaskGraphNodeID addToGraph(
        TaskGraphBuilder &builder, Span<const TaskGraphNodeID> deps)
    {
        return mwGPU::pushBuiltin(builder, deps, mb2::NodeRecycleEntities);
    }
};

class SortArchetypeNodeBase : public NodeBase {
public:
    static inline TaskGraphNodeID addToGraph(
        TaskGraphBuilder &builder, Span<const TaskGraphNodeID> deps,
        uint32_t archetype_id, int32_t component_id)
    {
        return mwGPU::pushBuiltin(builder, deps, mb2::NodeSortArchetype,
                                  archetype_id, (uint32_t)component_id);
    }
};

template <typename ArchetypeT, typename ComponentT>
class SortArchetypeNode : public SortArchetypeNodeBase {
public:
    static inline TaskGraphNodeID addToGraph(
        TaskGraphBuilder &builder, Span<const TaskGraphNodeID> deps)
    {
        return SortArchetypeNodeBase::addToGraph(builder, deps,
            TypeTracker::typeID<ArchetypeT>(), (int32_t)TypeTracker::typeID<ComponentT>());
    }
};

template <typename ArchetypeT>
class CompactArchetypeNode : public NodeBase {
public:
    static inline TaskGraphNodeID addToGraph(
        TaskGraphBuilder &builder, Span<const TaskGraphNodeID> deps)
    {
        return mwGPU::pushBuiltin(builder, deps, mb2::NodeCompactArchetype,
                                  TypeTracker::typeID<ArchetypeT>(), 1u);
    }
};

}
