#include "sim.hpp"

#ifdef MADRONA_GPU_MODE
#include <madrona/mw_gpu_entry.hpp>
#endif

using namespace madrona;
using namespace madrona::math;
using namespace madrona::phys;

namespace triggers {

constexpr float kDeltaT = 0.04f;
constexpr float kHalf = 6.f;           // walls' inner faces at +-6
constexpr float kWallThick = 0.5f;
constexpr float kWallHeight = 2.f;
constexpr float kAgentStep = 0.35f;
constexpr float kAgentReach = 5.f;
constexpr float kPickupScale = 0.6f;

// the zone the per-world system queries
static inline AABB zoneBox()
{
    return AABB { Vector3 { -1.5f, -1.5f, 0.f }, Vector3 { 1.5f, 1.5f, 2.f } };
}

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    base::registerTypes(registry);
    PhysicsSystem::registerTypes(registry);

    registry.registerComponent<Kind>();
    registry.registerComponent<Action>();
    registry.registerComponent<Touched>();

    registry.registerSingleton<PairObs>();
    registry.registerSingleton<ZoneObs>();

    registry.registerArchetype<Agent>(
        ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumAgents);
    registry.registerArchetype<Prop>(
        ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumProps);
    registry.registerArchetype<Pickup>();

    registry.exportColumn<Agent, Action>((uint32_t)ExportID::Action);
    registry.exportSingleton<PairObs>((uint32_t)ExportID::Pairs);
    registry.exportSingleton<ZoneObs>((uint32_t)ExportID::Zone);
    registry.exportColumn<Agent, Position>((uint32_t)ExportID::AgentPos);
    registry.exportColumn<Pickup, Entity>((uint32_t)ExportID::PickupEntity);
    registry.exportColumn<Pickup, Position>((uint32_t)ExportID::PickupPos);
    registry.exportColumn<Prop, Entity>((uint32_t)ExportID::PropEntity);
}

// yaw by multiples of 45 degrees: (cos(a/2), 0, 0, sin(a/2)) as literals
static inline Quat yawQuat(int32_t eighth)
{
    constexpr float c = 0.92387953f, s = 0.38268343f, d = 0.70710678f;
    switch (eighth & 7) {
    case 0: return Quat { 1, 0, 0, 0 };
    case 1: return Quat { c, 0, 0, s };
    case 2: return Quat { d, 0, 0, d };
    case 3: return Quat { s, 0, 0, c };
    case 4: return Quat { 0, 0, 0, 1 };
    case 5: return Quat { -s, 0, 0, c };
    case 6: return Quat { -d, 0, 0, d };
    default: return Quat { -c, 0, 0, s };
    }
}

template <typename ArchetypeT>
static inline Entity makeBody(Engine &ctx, Vector3 pos, Quat rot, Diag3x3 scale,
                              SimObject obj, ResponseType resp, Kind kind)
{
    Entity e = ctx.makeEntity<ArchetypeT>();
    ctx.get<Position>(e) = pos;
    ctx.get<Rotation>(e) = rot;
    ctx.get<Scale>(e) = scale;
    ctx.get<ObjectID>(e) = ObjectID { (int32_t)obj };
    ctx.get<ResponseType>(e) = resp;
    ctx.get<Velocity>(e) = Velocity { Vector3::zero(), Vector3::zero() };
    ctx.get<ExternalForce>(e) = Vector3::zero();
    ctx.get<ExternalTorque>(e) = Vector3::zero();
    ctx.get<Kind>(e) = kind;
    return e;
}

static inline Entity makePickup(Engine &ctx)
{
    RNG &rng = ctx.data().rng;
    float x = (rng.sampleUniform() - 0.5f) * 2.f * kAgentReach;
    float y = (rng.sampleUniform() - 0.5f) * 2.f * kAgentReach;
    Entity e = makeBody<Pickup>(ctx, Vector3 { x, y, 0.5f * kPickupScale }, Quat { 1, 0, 0, 0 },
                                Diag3x3 { kPickupScale, kPickupScale, kPickupScale },
                                SimObject::Pickup, ResponseType::Static, Kind::Pickup);
    ctx.get<Touched>(e).v = 0;
    return e;
}

// (Re)build the broadphase leaves of every body, in one fixed order
static void registerAll(Engine &ctx)
{
    Sim &sim = ctx.data();
    PhysicsSystem::reset(ctx);
    auto reg = [&](Entity e) {
        ctx.get<broadphase::LeafID>(e) =
            PhysicsSystem::registerEntity(ctx, e, ctx.get<ObjectID>(e));
    };
    reg(sim.floor);
    for (int32_t i = 0; i < kNumWalls; i++) reg(sim.walls[i]);
    for (int32_t i = 0; i < kNumAgents; i++) reg(sim.agents[i]);
    reg(sim.dumbbell);
    reg(sim.ball);
    for (int32_t i = 0; i < kNumPickups; i++) reg(sim.pickups[i]);
}

// a square loop of half size `half` around the origin, 8 steps per side
static inline Vector3 loopPos(int32_t step, float half, float z)
{
    const int32_t p = step & 31;
    const int32_t side = p / 8;
    const float f = (float)(p % 8) * 0.125f;
    const float a = -half + 2.f * half * f;
    switch (side) {
    case 0: return Vector3 { a, -half, z };
    case 1: return Vector3 { half, a, z };
    case 2: return Vector3 { -a, half, z };
    default: return Vector3 { -half, -a, z };
    }
}

// the ball goes back and forth along the diagonal, through the zone
static inline Vector3 ballPos(int32_t step)
{
    const int32_t p = step % 40;
    const float f = (float)(p < 20 ? p : 40 - p) * 0.05f;
    const float a = -4.f + 8.f * f;
    return Vector3 { a, a, 0.5f };
}

inline void agentMoveSystem(Engine &, Action &action, Position &pos)
{
    float x = pos.x + (float)(action.dx - 1) * kAgentStep;
    float y = pos.y + (float)(action.dy - 1) * kAgentStep;
    pos.x = x < -kAgentReach ? -kAgentReach : (x > kAgentReach ? kAgentReach : x);
    pos.y = y < -kAgentReach ? -kAgentReach : (y > kAgentReach ? kAgentReach : y);
}

inline void pathSystem(Engine &ctx, ZoneObs &zone)
{
    Sim &sim = ctx.data();
    sim.step += 1;
    zone.step = sim.step;
    ctx.get<Position>(sim.dumbbell) = loopPos(sim.step, 2.f, 0.6f);
    ctx.get<Rotation>(sim.dumbbell) = yawQuat(sim.step / 3);
    ctx.get<Position>(sim.ball) = ballPos(sim.step);
}

// per CandidateCollision row: idempotent flags only (rows run in any order)
inline void touchSystem(Engine &ctx, CandidateCollision &c)
{
    const Kind ka = ctx.get<Kind>(c.a);
    const Kind kb = ctx.get<Kind>(c.b);
    const bool a_touches = ka == Kind::Agent || ka == Kind::Dumbbell;
    const bool b_touches = kb == Kind::Agent || kb == Kind::Dumbbell;
    if (ka == Kind::Pickup && b_touches) ctx.get<Touched>(c.a).v = 1;
    if (kb == Kind::Pickup && a_touches) ctx.get<Touched>(c.b).v = 1;
}

inline void pairSystem(Engine &ctx, PairObs &obs)
{
    obs.count = 0;
    for (int32_t i = 0; i < kMaxPairs; i++) {
        for (int32_t j = 0; j < 4; j++) obs.pairs[i][j] = -1;
    }
    ctx.iterateQuery(ctx.data().candQuery, [&](CandidateCollision &c) {
        if (obs.count < kMaxPairs) {
            // column 0 of every table is the Entity (both backends)
            obs.pairs[obs.count][0] = ctx.getDirect<Entity>(0, c.a).id;
            obs.pairs[obs.count][1] = ctx.getDirect<Entity>(0, c.b).id;
            obs.pairs[obs.count][2] = (int32_t)c.aPrim;
            obs.pairs[obs.count][3] = (int32_t)c.bPrim;
        }
        obs.count += 1;
    });
}

inline void zoneSystem(Engine &ctx, ZoneObs &zone)
{
    Sim &sim = ctx.data();
    const AABB box = zoneBox();
    zone.numFound = 0;
    zone.firstFound = -1;
    PhysicsSystem::findEntitiesWithinAABB(ctx, box, [&](Entity e) {
        if (zone.numFound == 0) zone.firstFound = e.id;
        zone.numFound += 1;
    });
    zone.agentInZone = PhysicsSystem::checkEntityAABBOverlap(ctx, box, sim.agents[0]) ? 1 : 0;
    zone.dumbbellInZone = PhysicsSystem::checkEntityAABBOverlap(ctx, box, sim.dumbbell) ? 1 : 0;
    zone.ballInZone = PhysicsSystem::checkEntityAABBOverlap(ctx, box, sim.ball) ? 1 : 0;
    const Vector3 b = ctx.get<Position>(sim.ball);
    zone.ballCentreInZone = (b.x > box.pMin.x && b.x < box.pMax.x &&
                             b.y > box.pMin.y && b.y < box.pMax.y) ? 1 : 0;

    // replace the pickups an agent or the dumbbell overlapped this step
    bool replaced = false;
    for (int32_t i = 0; i < kNumPickups; i++) {
        if (ctx.get<Touched>(sim.pickups[i]).v == 0) continue;
        ctx.destroyEntity(sim.pickups[i]);
        sim.pickups[i] = makePickup(ctx);
        zone.respawns += 1;
        replaced = true;
    }
    if (replaced) registerAll(ctx);
}

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);

    auto move = builder.addToGraph<ParallelForNode<Engine, agentMoveSystem,
        Action, Position>>({});
    auto path = builder.addToGraph<ParallelForNode<Engine, pathSystem,
        ZoneObs>>({move});

    auto broadphase = PhysicsSystem::setupBroadphaseTasks(builder, {path});
    auto overlaps = PhysicsSystem::setupStandaloneBroadphaseOverlapTasks(builder, {broadphase});
#ifdef TRIGGERS_WITH_SOLVER
    // build variant (GPU only): the overlap rows and a solver step in one graph, which the
    // engine rejects when the launch graph is built
    overlaps = PhysicsSystem::setupPhysicsStepTasks(builder, {overlaps}, 1);
#endif

    auto touch = builder.addToGraph<ParallelForNode<Engine, touchSystem,
        CandidateCollision>>({overlaps});
    auto pairs = builder.addToGraph<ParallelForNode<Engine, pairSystem,
        PairObs>>({touch});
    auto zone = builder.addToGraph<ParallelForNode<Engine, zoneSystem,
        ZoneObs>>({pairs});

    auto cleanup = PhysicsSystem::setupStandaloneBroadphaseCleanupTasks(builder, {zone});
    auto compact = builder.addToGraph<CompactArchetypeNode<Pickup>>({cleanup});
#ifdef MADRONA_GPU_MODE
    builder.addToGraph<RecycleEntitiesNode>({compact});
#else
    (void)compact;
#endif
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx),
      rng(init.seed),
      step(0)
{
    PhysicsSystem::init(ctx, cfg.objMgr, kDeltaT, 1, -9.8f * math::up, kMaxBodies);

    const Quat upright { 1, 0, 0, 0 };
    floor = makeBody<Prop>(ctx, Vector3 { 0, 0, 0 }, upright, Diag3x3 { 1, 1, 1 },
                           SimObject::Floor, ResponseType::Static, Kind::Floor);
    const float reach = kHalf + kWallThick;
    const float mid = kHalf + 0.5f * kWallThick;
    const float hz = 0.5f * kWallHeight;
    walls[0] = makeBody<Prop>(ctx, Vector3 { 0, -mid, hz }, upright,
                              Diag3x3 { 2.f * reach, kWallThick, kWallHeight },
                              SimObject::Wall, ResponseType::Static, Kind::Wall);
    walls[1] = makeBody<Prop>(ctx, Vector3 { 0, mid, hz }, upright,
                              Diag3x3 { 2.f * reach, kWallThick, kWallHeight },
                              SimObject::Wall, ResponseType::Static, Kind::Wall);
    walls[2] = makeBody<Prop>(ctx, Vector3 { -mid, 0, hz }, upright,
                              Diag3x3 { kWallThick, 2.f * kHalf, kWallHeight },
                              SimObject::Wall, ResponseType::Static, Kind::Wall);
    walls[3] = makeBody<Prop>(ctx, Vector3 { mid, 0, hz }, upright,
                              Diag3x3 { kWallThick, 2.f * kHalf, kWallHeight },
                              SimObject::Wall, ResponseType::Static, Kind::Wall);
    dumbbell = makeBody<Prop>(ctx, loopPos(0, 2.f, 0.6f), upright, Diag3x3 { 1, 1, 1 },
                              SimObject::Dumbbell, ResponseType::Kinematic, Kind::Dumbbell);
    ball = makeBody<Prop>(ctx, ballPos(0), upright, Diag3x3 { 1, 1, 1 },
                          SimObject::Ball, ResponseType::Kinematic, Kind::Ball);
    for (int32_t i = 0; i < kNumAgents; i++) {
        float x = (rng.sampleUniform() - 0.5f) * 2.f * kAgentReach;
        float y = (rng.sampleUniform() - 0.5f) * 2.f * kAgentReach;
        agents[i] = makeBody<Agent>(ctx, Vector3 { x, y, 0.75f }, upright,
                                    Diag3x3 { 0.8f, 0.8f, 1.5f }, SimObject::Agent,
                                    ResponseType::Kinematic, Kind::Agent);
        ctx.get<Action>(agents[i]) = Action { 1, 1 };
    }
    for (int32_t i = 0; i < kNumPickups; i++) pickups[i] = makePickup(ctx);
    registerAll(ctx);
    candQuery = ctx.query<CandidateCollision>();

    PairObs &obs = ctx.singleton<PairObs>();
    obs.count = 0;
    for (int32_t i = 0; i < kMaxPairs; i++) {
        for (int32_t j = 0; j < 4; j++) obs.pairs[i][j] = -1;
    }
    ZoneObs &zone = ctx.singleton<ZoneObs>();
    zone = ZoneObs { 0, -1, 0, 0, 0, 0, 0, 0 };
}

}

#ifdef MADRONA_GPU_MODE
MADRONA_BUILD_MWGPU_ENTRY(triggers::Engine, triggers::Sim, triggers::Config, triggers::WorldInit);
#endif
