#include "sim.hpp"

#ifdef MADRONA_GPU_MODE
#include <madrona/mw_gpu_entry.hpp>
#endif

using namespace madrona;
using namespace madrona::math;
using namespace madrona::phys;

namespace crowd {

constexpr float kDeltaT = 0.04f;
constexpr CountT kNumSubsteps = 4;
constexpr float kWallThick = 0.5f;
constexpr float kWallHeight = 6.f;
constexpr float kCell = 2.f;               // pen area per dynamic body: one kCell x kCell cell

// bodies per world (plane and walls included), chosen per world and episode: below, at and
// above the engine's 128-body warp-per-world path
static constexpr int32_t kEpisodeSizes[kNumEpisodeSizes] = { 20, 128, 129, 200, 300, 700, 1500 };
static_assert(kEpisodeSizes[kNumEpisodeSizes - 1] == kVariedMaxBodies);

// the objects of the crowd, in turn
static constexpr SimObject kKinds[] = {
    SimObject::Box, SimObject::Ball, SimObject::Wedge, SimObject::PentaPyramid, SimObject::Ball,
};
constexpr int32_t kNumKinds = sizeof(kKinds) / sizeof(kKinds[0]);

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    base::registerTypes(registry);
    PhysicsSystem::registerTypes(registry);

    registry.registerSingleton<BodyCount>();
    registry.registerArchetype<Body>();

    registry.exportColumn<Body, Position>((uint32_t)ExportID::BodyPos);
    registry.exportColumn<Body, Rotation>((uint32_t)ExportID::BodyRot);
    registry.exportColumn<Body, Velocity>((uint32_t)ExportID::BodyVel);
    registry.exportColumn<Body, Entity>((uint32_t)ExportID::BodyEntity);
    registry.exportSingleton<BodyCount>((uint32_t)ExportID::BodyCount);
#ifdef CROWD_TWO_ARCHETYPES
    registry.registerArchetype<Body2>();
    registry.exportColumn<Body2, Position>((uint32_t)ExportID::Body2Pos);
    registry.exportColumn<Body2, Rotation>((uint32_t)ExportID::Body2Rot);
    registry.exportColumn<Body2, Velocity>((uint32_t)ExportID::Body2Vel);
    registry.exportColumn<Body2, Entity>((uint32_t)ExportID::Body2Entity);
#endif
}

template <typename ArchetypeT = Body>
static inline Entity makeBody(Engine &ctx, Vector3 pos, Quat rot, Diag3x3 scale,
                              SimObject obj, ResponseType resp, Vector3 lin_vel)
{
    Entity e = ctx.makeEntity<ArchetypeT>();
    ObjectID obj_id { (int32_t)obj };
    ctx.get<Position>(e) = pos;
    ctx.get<Rotation>(e) = rot;
    ctx.get<Scale>(e) = scale;
    ctx.get<ObjectID>(e) = obj_id;
    ctx.get<ResponseType>(e) = resp;
    ctx.get<Velocity>(e) = Velocity { lin_vel, Vector3::zero() };
    ctx.get<ExternalForce>(e) = Vector3::zero();
    ctx.get<ExternalTorque>(e) = Vector3::zero();
    ctx.get<broadphase::LeafID>(e) = PhysicsSystem::registerEntity(ctx, e, obj_id);
    return e;
}

// any orientation: four uniform samples, normalised
static inline Quat randomQuat(RNG &rng)
{
    float w = rng.sampleUniform() - 0.5f;
    float x = rng.sampleUniform() - 0.5f;
    float y = rng.sampleUniform() - 0.5f;
    float z = rng.sampleUniform() - 0.5f;
    return Quat { w, x, y, z }.normalize();
}

static int32_t episodeBodies(const Sim &sim)
{
    if (sim.uniformBodies != 0) return (int32_t)sim.uniformBodies;
    return kEpisodeSizes[(sim.seed + 3u * sim.episode) % (uint32_t)kNumEpisodeSizes];
}

// Reset the broadphase and create this episode's bodies (the previous ones were destroyed
// by the caller); one random sample per statement (argument evaluation order is unspecified)
static void spawnWorld(Engine &ctx)
{
    Sim &sim = ctx.data();
    RNG &rng = sim.rng;
    PhysicsSystem::reset(ctx);

    const int32_t total = episodeBodies(sim);
    const int32_t num_dyn = total - kNumStatic;
    int32_t side = 1;
    while (side * side < num_dyn) side++;
    const float pen = 0.5f * kCell * (float)side;     // pen interior: [-pen, pen]^2
    const Quat upright { 1, 0, 0, 0 };
    const Vector3 still = Vector3::zero();

    int32_t n = 0;
    sim.bodies[n++] = makeBody(ctx, Vector3 { 0, 0, 0 }, upright, Diag3x3 { 1, 1, 1 }, SimObject::Plane,
                               ResponseType::Static, still);
    const float reach = pen + kWallThick;
    const float mid = pen + 0.5f * kWallThick;
    sim.bodies[n++] = makeBody(ctx, Vector3 { 0, -mid, 0.5f * kWallHeight }, upright,
                               Diag3x3 { 2.f * reach, kWallThick, kWallHeight }, SimObject::Wall,
                               ResponseType::Static, still);
    sim.bodies[n++] = makeBody(ctx, Vector3 { 0, mid, 0.5f * kWallHeight }, upright,
                               Diag3x3 { 2.f * reach, kWallThick, kWallHeight }, SimObject::Wall,
                               ResponseType::Static, still);
    sim.bodies[n++] = makeBody(ctx, Vector3 { -mid, 0, 0.5f * kWallHeight }, upright,
                               Diag3x3 { kWallThick, 2.f * pen, kWallHeight }, SimObject::Wall,
                               ResponseType::Static, still);
    sim.bodies[n++] = makeBody(ctx, Vector3 { mid, 0, 0.5f * kWallHeight }, upright,
                               Diag3x3 { kWallThick, 2.f * pen, kWallHeight }, SimObject::Wall,
                               ResponseType::Static, still);

    for (int32_t i = 0; i < num_dyn; i++) {
        const SimObject obj = kKinds[i % kNumKinds];
        Vector3 pos;
        Diag3x3 scale { 1.f, 1.f, 1.f };
        Vector3 vel = still;
        if ((Layout)sim.layout == Layout::Clustered) {
            // tiny boxes on a spiral that shrinks by 3/4 per body, along x, y and z in turn:
            // every midpoint split of the rebuild peels off a few leaves only
            float r = 0.5f * pen;
            for (int32_t k = 0; k < i; k++) r *= 0.75f;
            const int32_t axis = i % 3;
            pos = Vector3 { -0.5f * pen, -0.5f * pen, 1.f };
            if (axis == 0) pos.x += r;
            else if (axis == 1) pos.y += r;
            else pos.z += r;
            scale = Diag3x3 { 0.05f, 0.05f, 0.05f };
        } else {
            const int32_t gx = i % side, gy = i / side;
            pos.x = -pen + kCell * ((float)gx + 0.5f);
            pos.x += 0.6f * (rng.sampleUniform() - 0.5f);
            pos.y = -pen + kCell * ((float)gy + 0.5f);
            pos.y += 0.6f * (rng.sampleUniform() - 0.5f);
            pos.z = 0.8f + 1.5f * rng.sampleUniform();
            if (obj == SimObject::Ball) {
                const float s = 0.8f + 0.3f * rng.sampleUniform();
                scale = Diag3x3 { s, s, s };
            } else {
                scale.d0 = 0.7f + 0.4f * rng.sampleUniform();
                scale.d1 = 0.7f + 0.4f * rng.sampleUniform();
                scale.d2 = 0.7f + 0.4f * rng.sampleUniform();
            }
            vel.x = 6.f * (rng.sampleUniform() - 0.5f);
            vel.y = 6.f * (rng.sampleUniform() - 0.5f);
        }
        const Quat rot = obj == SimObject::Ball ? upright : randomQuat(rng);
#ifdef CROWD_TWO_ARCHETYPES
        if (i % kSecondEvery == kSecondEvery - 1) {
            sim.bodies[n++] = makeBody<Body2>(ctx, pos, rot, scale, obj, ResponseType::Dynamic, vel);
            continue;
        }
#endif
        sim.bodies[n++] = makeBody(ctx, pos, rot, scale, obj, ResponseType::Dynamic, vel);
    }
    sim.numBodies = n;
    ctx.singleton<BodyCount>().count = n;
#ifdef CROWD_TWO_ARCHETYPES
    ctx.singleton<BodyCount>().second = num_dyn / kSecondEvery;
#endif
}

// One invocation per world: at the end of an episode, destroy every body and respawn
inline void episodeSystem(Engine &ctx, BodyCount &)
{
    Sim &sim = ctx.data();
    sim.stepInEpisode += 1;
    if (sim.episodeLen == 0 || sim.stepInEpisode < sim.episodeLen) return;
    sim.stepInEpisode = 0;
    for (int32_t i = 0; i < sim.numBodies; i++) ctx.destroyEntity(sim.bodies[i]);
    sim.episode += 1;
    spawnWorld(ctx);
}

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);
    auto episode = builder.addToGraph<ParallelForNode<Engine, episodeSystem, BodyCount>>({});
    // destroyed bodies leave holes (CPU) / unsorted rows (GPU)
    auto compact = builder.addToGraph<CompactArchetypeNode<Body>>({episode});
#ifdef MADRONA_GPU_MODE
    auto post_reset = builder.addToGraph<RecycleEntitiesNode>({compact});
#else
    auto post_reset = compact;
#endif
    // a respawn re-registered every body: the broadphase rebuilds the tree
    auto broadphase = PhysicsSystem::setupBroadphaseTasks(builder, {post_reset});
    auto physics = PhysicsSystem::setupPhysicsStepTasks(builder, {broadphase}, kNumSubsteps);
    PhysicsSystem::setupCleanupTasks(builder, {physics});
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx),
      rng(init.seed),
      seed(init.seed),
      episodeLen(cfg.episodeLen),
      uniformBodies(cfg.uniformBodies),
      layout(cfg.layout),
      stepInEpisode(0),
      episode(0),
      numBodies(0)
{
    PhysicsSystem::init(ctx, cfg.objMgr, kDeltaT, kNumSubsteps, -9.8f * math::up,
                        cfg.uniformBodies != 0 ? (CountT)cfg.uniformBodies : (CountT)kVariedMaxBodies);
    spawnWorld(ctx);
}

}

#ifdef MADRONA_GPU_MODE
MADRONA_BUILD_MWGPU_ENTRY(crowd::Engine, crowd::Sim, crowd::Config, crowd::WorldInit);
#endif
