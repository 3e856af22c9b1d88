#include "sim.hpp"
#include <madrona/mw_gpu_entry.hpp>

using namespace madrona;

namespace sortsweep {

template <typename T>
static inline void fillPayload(T &p, uint32_t world, uint32_t uid, uint32_t c)
{
    for (uint32_t i = 0; i < (uint32_t)sizeof(p.b); i++) p.b[i] = payloadByte(world, uid, c, i);
}

template <typename T>
static inline uint32_t payloadMismatch(const T &p, uint32_t world, uint32_t uid, uint32_t c)
{
    for (uint32_t i = 0; i < (uint32_t)sizeof(p.b); i++) {
        if (p.b[i] != payloadByte(world, uid, c, i)) return 1u << (3 + c);
    }
    return 0;
}

// the step whose keys the rows hold: rekeyed every step, or keyed once at creation
static inline uint32_t keyStep(Engine &ctx)
{
    return ctx.data().shape == ShapeChurn ? 0u : ctx.singleton<StepCounter>().t;
}

static inline void makeItem(Engine &ctx, uint32_t t)
{
    Sim &sim = ctx.data();
    const uint32_t world = (uint32_t)ctx.worldID().idx;
    const uint32_t uid = sim.nextUid++;
    Entity e = ctx.makeEntity<Item>();
    if (e.id < 0) return;
    const uint32_t key = keyOf(sim.seed, uid, sim.shape == ShapeChurn ? 0u : t, sim.keyMode);
    ctx.get<Uid>(e).v = uid;
    ctx.get<Key4>(e).v = key;
    ctx.get<Key8>(e) = Key8 { key, key8Hi(key, uid) };
    fillPayload(ctx.get<P1>(e), world, uid, 0);
    fillPayload(ctx.get<P2>(e), world, uid, 1);
    fillPayload(ctx.get<P3>(e), world, uid, 2);
    fillPayload(ctx.get<P5>(e), world, uid, 3);
    fillPayload(ctx.get<P8>(e), world, uid, 4);
    fillPayload(ctx.get<P12>(e), world, uid, 5);
    fillPayload(ctx.get<P20>(e), world, uid, 6);
    fillPayload(ctx.get<P24>(e), world, uid, 7);
    fillPayload(ctx.get<P32>(e), world, uid, 8);
    fillPayload(ctx.get<P48>(e), world, uid, 9);
    fillPayload(ctx.get<P6>(e), world, uid, 10);
    ctx.get<Check>(e).mismatch = 0;
}

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    registry.registerComponent<Uid>();
    registry.registerComponent<Key4>();
    registry.registerComponent<Key8>();
    registry.registerComponent<P1>();
    registry.registerComponent<P2>();
    registry.registerComponent<P3>();
    registry.registerComponent<P5>();
    registry.registerComponent<P8>();
    registry.registerComponent<P12>();
    registry.registerComponent<P20>();
    registry.registerComponent<P24>();
    registry.registerComponent<P32>();
    registry.registerComponent<P48>();
    registry.registerComponent<P6>();
    registry.registerComponent<Check>();
    registry.registerSingleton<StepCounter>();
    registry.registerSingleton<Summary>();
    registry.registerArchetype<Item>();
    // about half the payloads are exported (copied back after a sort); P1, P5, P6, P8,
    // P20, P32 and Key8 are not (their buffers are flipped): both paths move 1-, 2-, 4-,
    // 8- and 16-byte units
    registry.exportColumn<Item, Entity>((uint32_t)ExportID::Entity);
    registry.exportColumn<Item, Uid>((uint32_t)ExportID::Uid);
    registry.exportColumn<Item, Key4>((uint32_t)ExportID::Key4);
    registry.exportColumn<Item, Check>((uint32_t)ExportID::Check);
    registry.exportColumn<Item, P2>((uint32_t)ExportID::P2);
    registry.exportColumn<Item, P3>((uint32_t)ExportID::P3);
    registry.exportColumn<Item, P12>((uint32_t)ExportID::P12);
    registry.exportColumn<Item, P24>((uint32_t)ExportID::P24);
    registry.exportColumn<Item, P48>((uint32_t)ExportID::P48);
    registry.exportSingleton<Summary>((uint32_t)ExportID::Summary);
}

inline void tickSystem(Engine &, StepCounter &c)
{
    c.t += 1;
}

inline void rekeySystem(Engine &ctx, Uid &uid, Key4 &k4, Key8 &k8)
{
    const uint32_t key = keyOf(ctx.data().seed, uid.v, ctx.singleton<StepCounter>().t, ctx.data().keyMode);
    k4.v = key;
    k8 = Key8 { key, key8Hi(key, uid.v) };
}

inline void destroySystem(Engine &ctx, Entity &e, Uid &uid)
{
    const Sim &sim = ctx.data();
    const uint32_t t = ctx.singleton<StepCounter>().t;
    if (t == sim.killStep || hashOf(sim.seed, uid.v, t) < sim.destroyThreshold) ctx.destroyEntity(e);
}

// one thread per world, so a world's new rows are appended in creation order
inline void createSystem(Engine &ctx, StepCounter &c)
{
    const Sim &sim = ctx.data();
    if (c.t == sim.killStep) return;
    for (uint32_t i = 0; i < sim.createsPerStep; i++) makeItem(ctx, c.t);
}

inline void checkSystem(Engine &ctx, Entity &e, Uid &uid, Key4 &k4, Key8 &k8,
                        P1 &p1, P2 &p2, P3 &p3, P5 &p5, P8 &p8, P12 &p12, P20 &p20,
                        P24 &p24, P32 &p32, P48 &p48, P6 &p6, Check &check)
{
    const uint32_t world = (uint32_t)ctx.worldID().idx;
    const uint32_t u = uid.v;
    uint32_t bad = 0;
    // the entity must resolve to this very row (a stale slot points elsewhere)
    const Loc l = ctx.loc(e);
    if (!l.valid() || l.archetype != TypeTracker::typeID<Item>() || &ctx.get<Uid>(l) != &uid) bad |= 1u;
    const uint32_t key = keyOf(ctx.data().seed, u, keyStep(ctx), ctx.data().keyMode);
    if (k4.v != key) bad |= 2u;
    if (k8.v != key || k8.hi != key8Hi(key, u)) bad |= 4u;
    bad |= payloadMismatch(p1, world, u, 0);
    bad |= payloadMismatch(p2, world, u, 1);
    bad |= payloadMismatch(p3, world, u, 2);
    bad |= payloadMismatch(p5, world, u, 3);
    bad |= payloadMismatch(p8, world, u, 4);
    bad |= payloadMismatch(p12, world, u, 5);
    bad |= payloadMismatch(p20, world, u, 6);
    bad |= payloadMismatch(p24, world, u, 7);
    bad |= payloadMismatch(p32, world, u, 8);
    bad |= payloadMismatch(p48, world, u, 9);
    bad |= payloadMismatch(p6, world, u, 10);
    check.mismatch = bad;
}

// walks the world's rows through worldOffsets / worldCounts
inline void summarySystem(Engine &ctx, Summary &s)
{
    uint32_t count = 0, hash = 0;
    auto q = ctx.query<Uid>();
    ctx.iterateQuery(q, [&](Uid &uid) {
        hash += summaryTerm(uid.v, count);
        count++;
    });
    s = Summary { count, hash };
}

void Sim::setupTasks(TaskGraphManager &mgr, const Config &cfg)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);
    TaskGraphNodeID last = builder.addToGraph<ParallelForNode<Engine, tickSystem, StepCounter>>({});
    if (cfg.shape != ShapeChurn) {
        last = builder.addToGraph<ParallelForNode<Engine, rekeySystem, Uid, Key4, Key8>>({last});
    }
    if (cfg.shape != ShapeSort) {
        last = builder.addToGraph<ParallelForNode<Engine, destroySystem, Entity, Uid>>({last});
        last = builder.addToGraph<ParallelForNode<Engine, createSystem, StepCounter>>({last});
    }
    if (cfg.shape != ShapeChurn) {
        last = cfg.sortOnKey8 ? builder.addToGraph<SortArchetypeNode<Item, Key8>>({last})
                              : builder.addToGraph<SortArchetypeNode<Item, Key4>>({last});
    }
    if (cfg.shape != ShapeSort) {
        last = builder.addToGraph<CompactArchetypeNode<Item>>({last});
        last = builder.addToGraph<RecycleEntitiesNode>({last});
    }
    last = builder.addToGraph<ParallelForNode<Engine, checkSystem, Entity, Uid, Key4, Key8,
        P1, P2, P3, P5, P8, P12, P20, P24, P32, P48, P6, Check>>({last});
    if (cfg.shape != ShapeSort) {
        builder.addToGraph<ParallelForNode<Engine, summarySystem, Summary>>({last});
    }
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx), seed(init.seed), nextUid(0), createsPerStep(init.createsPerStep),
      killStep(init.killStep), shape(cfg.shape), keyMode(cfg.keyMode),
      destroyThreshold(cfg.destroyThreshold)
{
    ctx.singleton<StepCounter>().t = 0;
    ctx.singleton<Summary>() = Summary { 0, 0 };
    for (uint32_t i = 0; i < init.initCount; i++) makeItem(ctx, 0);
}

}

MADRONA_BUILD_MWGPU_ENTRY(sortsweep::Engine, sortsweep::Sim, sortsweep::Config, sortsweep::WorldInit);
