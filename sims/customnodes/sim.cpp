#include "sim.hpp"

#ifdef MADRONA_GPU_MODE
#include <madrona/mw_gpu_entry.hpp>
#endif

using namespace madrona;

namespace customnodes {

#ifdef MADRONA_GPU_MODE
template <typename NodeT> using DataIDOf = TaskGraph::TypedDataID<NodeT>;
#else
template <typename NodeT> using DataIDOf = TaskGraphBuilder::TypedDataID<NodeT>;
#endif

constexpr uint32_t kTokenSalt = 0x5bd1e995u;
// CoopNode blocks per world, by step: includes steps with none
constexpr uint32_t kCoopPattern[8] = { 0, 3, 6, 1, 0, 5, 2, 6 };

static inline uint32_t mix32(uint32_t x)
{
    x ^= x >> 16;
    x *= 0x7feb352du;
    x ^= x >> 15;
    x *= 0x846ca68bu;
    x ^= x >> 16;
    return x;
}

static inline uint32_t tokenHash(Entity e, uint32_t v, uint32_t salt)
{
    return mix32(v ^ mix32((uint32_t)e.id * 2654435761u + e.gen + salt));
}

static inline uint32_t coopTerm(uint32_t salt, uint32_t step, uint32_t j, uint32_t t)
{
    return mix32(salt + step * 0x9e3779b9u + j * 0x85ebca6bu + t);
}

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    registry.registerComponent<TokenVal>();
    registry.registerComponent<TokenOut>();
    registry.registerSingleton<WorldSum>();
    registry.registerSingleton<CoopOut>();
    registry.registerSingleton<Census>();
    registry.registerArchetype<Token>();

    registry.exportSingleton<WorldSum>((uint32_t)ExportID::WorldSum);
    registry.exportSingleton<CoopOut>((uint32_t)ExportID::CoopOut);
    registry.exportSingleton<Census>((uint32_t)ExportID::Census);
    registry.exportColumn<Token, Entity>((uint32_t)ExportID::TokenEntity);
    registry.exportColumn<Token, TokenVal>((uint32_t)ExportID::TokenVal);
    registry.exportColumn<Token, TokenOut>((uint32_t)ExportID::TokenOut);

#ifdef CUSTOMNODES_PROBE
    registry.registerComponent<ProbeRec>();
    registry.registerSingleton<ProbeInfo>();
    registry.registerArchetype<ProbeSlot>(ComponentMetadataSelector<> {}, ArchetypeFlags::None, kProbeSlots);
    registry.exportColumn<ProbeSlot, ProbeRec>((uint32_t)ExportID::ProbeRec);
    registry.exportSingleton<ProbeInfo>((uint32_t)ExportID::ProbeInfo);
#endif
}

static inline void makeToken(Engine &ctx)
{
    Sim &sim = ctx.data();
    Entity e = ctx.makeEntity<Token>();
    ctx.get<TokenVal>(e).v = (uint32_t)sim.rng.sampleI32(0, 1 << 30);
    ctx.get<TokenOut>(e).h = 0;
    sim.tokens[sim.numTokens++] = e;
    sim.totalMade += 1;
}

// One world's churn: every token's value moves on, then tokens die and are born.
static void spawnWorld(Engine &ctx)
{
    Sim &sim = ctx.data();
    sim.curStep += 1;
    ctx.singleton<CoopOut>() = CoopOut {};
    for (int32_t i = 0; i < sim.numTokens; i++) {
        TokenVal &tv = ctx.get<TokenVal>(sim.tokens[i]);
        tv.v = tv.v * 1664525u + 1013904223u;
    }
    if (sim.empty) {
        return;
    }
    if (sim.curStep % 9 == 0) {
        for (int32_t i = 0; i < sim.numTokens; i++) {
            ctx.destroyEntity(sim.tokens[i]);
        }
        sim.numTokens = 0;
        return;
    }
    int32_t i = 0;
    while (i < sim.numTokens) {
        if (sim.rng.sampleI32(0, 4) == 0) {
            ctx.destroyEntity(sim.tokens[i]);
            sim.tokens[i] = sim.tokens[sim.numTokens - 1];
            sim.numTokens -= 1;
        } else {
            i += 1;
        }
    }
    const int32_t births = sim.rng.sampleI32(0, 5);
    for (int32_t b = 0; b < births && sim.numTokens < kMaxTokens; b++) {
        makeToken(ctx);
    }
}

inline void tokenRowSystem(Engine &, Entity &e, TokenVal &v, TokenOut &out)
{
    out.h = tokenHash(e, v.v, kTokenSalt);
}

struct SpawnNode : public NodeBase {
#ifdef MADRONA_GPU_MODE
    void run(int32_t world_idx)
    {
        Engine ctx = TaskGraph::makeContext<Engine>(WorldID { world_idx });
        spawnWorld(ctx);
    }
#else
    void cpuRun(Context &ctx, TaskGraph &) { spawnWorld(static_cast<Engine &>(ctx)); }
#endif
};

// Warp-per-world reduction over the world's rows of the (compacted) Token table.
struct WarpSumNode : public NodeBase {
    uint32_t tokenArchetype;
    uint32_t valComponent;

    WarpSumNode(uint32_t token_archetype, uint32_t val_component)
        : tokenArchetype(token_archetype), valComponent(val_component)
    {}

#ifdef MADRONA_GPU_MODE
    void run(int32_t world_idx)
    {
        StateManager *mgr = mwGPU::getStateManager();
        const int32_t lane = (int32_t)(threadIdx.x % 32);
        const int32_t off = mgr->getArchetypeWorldOffsets(tokenArchetype)[world_idx];
        const int32_t cnt = mgr->getArchetypeWorldCounts(tokenArchetype)[world_idx];
        const TokenVal *vals = (const TokenVal *)mgr->getArchetypeComponent(tokenArchetype, valComponent);
        const Entity *ents = (const Entity *)mgr->getArchetypeColumn(tokenArchetype, 0);
        uint32_t sum = 0, ids = 0, max_val = 0;
        for (int32_t r = lane; r < cnt; r += 32) {
            const uint32_t v = vals[off + r].v;
            sum += v;
            ids ^= (uint32_t)ents[off + r].id;
            max_val = v > max_val ? v : max_val;
        }
        for (int32_t m = 16; m > 0; m >>= 1) {
            sum += __shfl_xor_sync(0xffffffffu, sum, m);
            ids ^= __shfl_xor_sync(0xffffffffu, ids, m);
            const uint32_t o = __shfl_xor_sync(0xffffffffu, max_val, m);
            max_val = o > max_val ? o : max_val;
        }
        if (lane == 0) {
            Engine ctx = TaskGraph::makeContext<Engine>(WorldID { world_idx });
            ctx.singleton<WorldSum>() = WorldSum { (uint32_t)cnt, sum, ids, max_val };
        }
    }
#else
    void cpuRun(Context &base, TaskGraph &)
    {
        Engine &ctx = static_cast<Engine &>(base);
        WorldSum s {};
        auto q = ctx.query<Entity, TokenVal>();
        ctx.iterateQuery(q, [&](Entity &e, TokenVal &v) {
            s.count += 1;
            s.sum += v.v;
            s.xorIDs ^= (uint32_t)e.id;
            s.maxVal = v.v > s.maxVal ? v.v : s.maxVal;
        });
        ctx.singleton<WorldSum>() = s;
    }
#endif
};

// One invocation per Token row (addDynamicCountNode).
struct TokenRowsNode : public NodeBase {
    uint32_t salt;
    QueryRef *queryRef;

    TokenRowsNode(uint32_t salt_)
        : salt(salt_), queryRef(nullptr)
    {
#ifdef MADRONA_GPU_MODE
        queryRef = mwGPU::getStateManager()->query<Entity, TokenVal, TokenOut>().getSharedRef();
#endif
    }

#ifdef MADRONA_GPU_MODE
    uint32_t numInvocations()
    {
        return mwGPU::getStateManager()->numMatchingEntities(queryRef);
    }

    void run(int32_t invocation)
    {
        int32_t row = invocation;
        mwGPU::getStateManager()->iterateArchetypesRaw<3>(queryRef,
            [&](int32_t num_rows, WorldID *worlds, void *ents, void *vals, void *outs) {
                if (row >= num_rows) {
                    row -= num_rows;
                    return false;
                }
                if (worlds[row].idx >= 0) {
                    ((TokenOut *)outs)[row].h =
                        tokenHash(((Entity *)ents)[row], ((TokenVal *)vals)[row].v, salt);
                }
                return true;
            });
    }
#else
    void cpuRun(Context &base, TaskGraph &)
    {
        Engine &ctx = static_cast<Engine &>(base);
        auto q = ctx.query<Entity, TokenVal, TokenOut>();
        ctx.iterateQuery(q, [&](Entity &e, TokenVal &v, TokenOut &out) {
            out.h = tokenHash(e, v.v, salt);
        });
    }
#endif
};

// k blocks of 256 threads per world; each sums 256 terms through shared memory.
struct CoopNode : public NodeBase {
    uint32_t k;

#ifdef MADRONA_GPU_MODE
    void run(int32_t invocation)
    {
        __shared__ uint32_t partial[256];
        const uint32_t t = threadIdx.x;
        // the run keeps the count latched when it started
        if (invocation == 0 && t == 0) {
            numDynamicInvocations = 0;
        }
        const int32_t world_idx = invocation / (int32_t)k;
        const uint32_t j = (uint32_t)invocation % k;
        const Sim &sim = *(const Sim *)TaskGraph::getWorld(world_idx);
        partial[t] = coopTerm(sim.salt, sim.curStep, j, t);
        __syncthreads();
        for (uint32_t s = 128; s > 0; s >>= 1) {
            if (t < s) {
                partial[t] += partial[t + s];
            }
            __syncthreads();
        }
        if (t == 0) {
            Engine ctx = TaskGraph::makeContext<Engine>(WorldID { world_idx });
            CoopOut &out = ctx.singleton<CoopOut>();
            out.v[j] = partial[0];
            if (j == 0) {
                out.k = k;
            }
        }
        __syncthreads();
    }
#else
    void cpuRun(Context &base, TaskGraph &)
    {
        Engine &ctx = static_cast<Engine &>(base);
        const Sim &sim = ctx.data();
        CoopOut &out = ctx.singleton<CoopOut>();
        out.k = sim.coopK;
        for (uint32_t j = 0; j < sim.coopK; j++) {
            uint32_t sum = 0;
            for (uint32_t t = 0; t < 256; t++) {
                sum += coopTerm(sim.salt, sim.curStep, j, t);
            }
            out.v[j] = sum;
        }
    }
#endif
};

// Sets this step's CoopNode count (k per world) in the CoopNode's own data.
struct SetCountNode : public NodeBase {
    DataIDOf<CoopNode> target;
    uint32_t step;

    SetCountNode(DataIDOf<CoopNode> target_)
        : target(target_), step(0)
    {}

#ifdef MADRONA_GPU_MODE
    void run(int32_t)
    {
        step += 1;
        const uint32_t k = kCoopPattern[step % 8];
        CoopNode &coop = mwGPU::getTaskGraph(0).getNodeData(target);
        coop.k = k;
        coop.numDynamicInvocations = k * mwGPU::getStateManager()->numWorlds();
    }
#else
    void cpuRun(Context &ctx, TaskGraph &)
    {
        step += 1;
        static_cast<Engine &>(ctx).data().coopK = kCoopPattern[step % 8];
    }
#endif
};

struct CensusNode : public NodeBase {
#ifdef MADRONA_GPU_MODE
    void run(int32_t world_idx)
    {
        Engine ctx = TaskGraph::makeContext<Engine>(WorldID { world_idx });
        count(ctx);
    }
#else
    void cpuRun(Context &ctx, TaskGraph &) { count(static_cast<Engine &>(ctx)); }
#endif

    static void count(Engine &ctx)
    {
        Census &c = ctx.singleton<Census>();
        c.calls += 1;
        c.tokens = (uint32_t)ctx.data().numTokens;
        c.made = ctx.data().totalMade;
    }
};

#ifdef CUSTOMNODES_PROBE
// Invocation probe: every lane that runs invocation i reports into row i % kProbeSlots;
// the lanes of one warp that share an invocation report once, together.
struct ProbeNode : public NodeBase {
    uint32_t threads;
    uint32_t zeroOwnCount;

    ProbeNode(uint32_t threads_, uint32_t zero_own_count)
        : threads(threads_), zeroOwnCount(zero_own_count)
    {}

    void run(int32_t invocation)
    {
        const uint32_t lane = threadIdx.x % threads;
        if (zeroOwnCount && invocation == 0 && lane == 0) {
            numDynamicInvocations = 0;
        }
        StateManager *mgr = mwGPU::getStateManager();
        ProbeRec *recs = (ProbeRec *)mgr->getArchetypeComponent(
            TypeTracker::typeID<ProbeSlot>(), TypeTracker::typeID<ProbeRec>());
        ProbeRec &rec = recs[invocation % kProbeSlots];
        const unsigned peers = __match_any_sync(__activemask(), invocation);
        const uint32_t n = (uint32_t)__popc(peers);
        const uint32_t lane_sum = __reduce_add_sync(peers, lane);
        const uint32_t bits = __reduce_or_sync(peers, 1u << (lane % 32));
        if ((int)(threadIdx.x % 32) == __ffs(peers) - 1) {
            atomicAdd(&rec.hits, n);
            atomicAdd(&rec.invSum, (unsigned long long)invocation * n);
            atomicAdd(&rec.laneSum, (unsigned long long)lane_sum);
            atomicOr(&rec.lanes[lane / 32], bits);
            Engine ctx = TaskGraph::makeContext<Engine>(WorldID { 0 });
            atomicMax(&ctx.singleton<ProbeInfo>().maxInvPlus1, (uint32_t)invocation + 1);
        }
    }
};

struct ProbeCountNode : public NodeBase {
    DataIDOf<ProbeNode> target;
    uint32_t count;

    ProbeCountNode(uint32_t count_) : target { { -1 } }, count(count_) {}

    void run(int32_t)
    {
        mwGPU::getTaskGraph(0).getNodeData(target).numDynamicInvocations = count;
    }
};

struct FillerNode : public NodeBase {
    uint32_t v;
    FillerNode(uint32_t v_) : v(v_) {}
};

static void setupProbe(TaskGraphManager &mgr, const Config &cfg)
{
    TaskGraphBuilder &b = mgr.init(TaskGraphID::Step);
    for (uint32_t i = 0; i < cfg.extraNodeDatas; i++) {
        b.constructNodeData<FillerNode>(i);
    }
    auto probe_data = b.constructNodeData<ProbeNode>(cfg.probeThreads, cfg.probeDynamic);
    if (cfg.probeDynamic) {
        auto set_data = b.constructNodeData<ProbeCountNode>(cfg.probeCount);
        auto set = b.addNodeFn<&ProbeCountNode::run>(set_data, {}, Optional<TaskGraphNodeID>::none(), 1);
        b.addNodeFn<&ProbeNode::run>(probe_data, { set }, Optional<TaskGraphNodeID>::none(), 0,
                                     cfg.probeThreads);
        // the target's data ID goes in after the target node was added
        b.getDataRef(set_data).target = probe_data;
    } else {
        b.addNodeFn<&ProbeNode::run>(probe_data, {}, Optional<TaskGraphNodeID>::none(), cfg.probeCount,
                                     cfg.probeThreads);
    }
}
#endif

void Sim::setupTasks(TaskGraphManager &mgr, const Config &cfg)
{
    (void)cfg;
#ifdef MADRONA_GPU_MODE
#ifdef CUSTOMNODES_PROBE
    setupProbe(mgr, cfg);
#else
    const uint32_t num_worlds = mwGPU::getStateManager()->numWorlds();
    const auto none = Optional<TaskGraphNodeID>::none();

    TaskGraphBuilder &b = mgr.init(TaskGraphID::Step);
    auto spawn = b.addNodeFn<&SpawnNode::run>(b.constructNodeData<SpawnNode>(), {}, none, num_worlds, 1);
    auto compact = b.addToGraph<CompactArchetypeNode<Token>>({ spawn });
    // three branches
    b.addNodeFn<&WarpSumNode::run>(
        b.constructNodeData<WarpSumNode>(TypeTracker::typeID<Token>(), TypeTracker::typeID<TokenVal>()),
        { compact }, none, num_worlds, 32);
    auto rows = b.addDynamicCountNode<TokenRowsNode>({ compact }, 1, kTokenSalt);
#ifdef CUSTOMNODES_BENCH
    b.addToGraph<ParallelForNode<Engine, tokenRowSystem, Entity, TokenVal, TokenOut>>({ rows });
#else
    (void)rows;
#endif
    auto coop_data = b.constructNodeData<CoopNode>();
    auto setter = b.addOneOffNode<SetCountNode, 1>({ compact }, coop_data);
    b.addNodeFn<&CoopNode::run>(coop_data, { compact }, setter, 0, 256);

    TaskGraphBuilder &census = mgr.init(TaskGraphID::Census);
    census.addNodeFn<&CensusNode::run>(census.constructNodeData<CensusNode>(), {}, none, num_worlds, 1);
#endif
#else
    TaskGraphBuilder &b = mgr.init(TaskGraphID::Step);
    auto spawn = b.addNodeFn<&SpawnNode::cpuRun>(b.constructNodeData<SpawnNode>(), {});
    auto compact = b.addToGraph<CompactArchetypeNode<Token>>({ spawn });
    b.addNodeFn<&WarpSumNode::cpuRun>(
        b.constructNodeData<WarpSumNode>(TypeTracker::typeID<Token>(), TypeTracker::typeID<TokenVal>()),
        { compact });
    b.addNodeFn<&TokenRowsNode::cpuRun>(b.constructNodeData<TokenRowsNode>(kTokenSalt), { compact });
    auto coop_data = b.constructNodeData<CoopNode>();
    auto setter = b.addNodeFn<&SetCountNode::cpuRun>(b.constructNodeData<SetCountNode>(coop_data), { compact });
    b.addNodeFn<&CoopNode::cpuRun>(coop_data, { compact, setter }, setter);

    TaskGraphBuilder &census = mgr.init(TaskGraphID::Census);
    census.addNodeFn<&CensusNode::cpuRun>(census.constructNodeData<CensusNode>(), {});
#endif
}

Sim::Sim(Engine &ctx, const Config &, const WorldInit &init)
    : WorldBase(ctx),
      rng(init.seed),
      numTokens(0),
      empty(init.empty),
      salt(mix32(init.seed * 747796405u + 1u)),
      curStep(0),
      totalMade(0),
      coopK(0)
{
    ctx.singleton<WorldSum>() = WorldSum {};
    ctx.singleton<CoopOut>() = CoopOut {};
    if (!empty) {
        const int32_t n = 3 + rng.sampleI32(0, 6);
        for (int32_t i = 0; i < n; i++) {
            makeToken(ctx);
        }
    }
    ctx.singleton<Census>() = Census { 0, (uint32_t)numTokens, totalMade, 0 };
#ifdef CUSTOMNODES_PROBE
    ctx.singleton<ProbeInfo>() = ProbeInfo {};
    for (int32_t i = 0; i < kProbeSlots; i++) {
        Entity e = ctx.makeEntity<ProbeSlot>();
        ctx.get<ProbeRec>(e) = ProbeRec {};
    }
#endif
}

}

#ifdef MADRONA_GPU_MODE
MADRONA_BUILD_MWGPU_ENTRY(customnodes::Engine, customnodes::Sim,
                          customnodes::Config, customnodes::WorldInit);
#endif
