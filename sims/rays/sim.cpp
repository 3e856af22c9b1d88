#include "sim.hpp"

#ifdef MADRONA_GPU_MODE
#include <madrona/mw_gpu_entry.hpp>
#endif

using namespace madrona;
using namespace madrona::math;
using namespace madrona::phys;

namespace rays {

constexpr float kDeltaT = 0.04f;
constexpr CountT kNumSubsteps = 4;
constexpr float kWallThick = 0.5f;
constexpr float kWallHeight = 6.f;
constexpr float kCell = 2.f;               // pen area per dynamic body: one kCell x kCell cell

#ifdef RAYS_SPHERES
static constexpr SimObject kKinds[] = {
    SimObject::Box, SimObject::Ball, SimObject::Wedge, SimObject::Dumbbell, SimObject::OctPrism,
    SimObject::Ball, SimObject::PentaPyramid,
};
#else
static constexpr SimObject kKinds[] = {
    SimObject::Box, SimObject::Wedge, SimObject::Dumbbell, SimObject::OctPrism, SimObject::PentaPyramid,
};
#endif
constexpr int32_t kNumKinds = sizeof(kKinds) / sizeof(kKinds[0]);

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    base::registerTypes(registry);
    PhysicsSystem::registerTypes(registry);

    registry.registerComponent<RayOrigin>();
    registry.registerComponent<RayDir>();
    registry.registerComponent<RayMaxT>();
    registry.registerComponent<HitEntity>();
    registry.registerComponent<HitT>();
    registry.registerComponent<HitNormal>();
    registry.registerComponent<RayState>();
    registry.registerSingleton<BodyCount>();
    registry.registerArchetype<RayProbe>(ComponentMetadataSelector<> {}, ArchetypeFlags::None, kRaysPerWorld);
    registry.registerArchetype<Body>();

    registry.exportColumn<RayProbe, RayOrigin>((uint32_t)ExportID::RayOrigin);
    registry.exportColumn<RayProbe, RayDir>((uint32_t)ExportID::RayDir);
    registry.exportColumn<RayProbe, RayMaxT>((uint32_t)ExportID::RayMaxT);
    registry.exportColumn<RayProbe, HitEntity>((uint32_t)ExportID::HitEntity);
    registry.exportColumn<RayProbe, HitT>((uint32_t)ExportID::HitT);
    registry.exportColumn<RayProbe, HitNormal>((uint32_t)ExportID::HitNormal);
    registry.exportSingleton<BodyCount>((uint32_t)ExportID::BodyCount);
    registry.exportColumn<Body, Position>((uint32_t)ExportID::BodyPos);
    registry.exportColumn<Body, Entity>((uint32_t)ExportID::BodyEntity);
}

static inline Entity makeBody(Engine &ctx, Vector3 pos, Quat rot, Diag3x3 scale, SimObject obj,
                              ResponseType resp, Vector3 lin_vel)
{
    Entity e = ctx.makeEntity<Body>();
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
    return 8 + (int32_t)((sim.seed * 7u + 13u * sim.episode) % (sim.variedBodies - 7u));
}

// Reset the broadphase and create this episode's bodies (the previous ones were destroyed by
// the caller); one random sample per statement (argument evaluation order is unspecified)
static void spawnWorld(Engine &ctx)
{
    Sim &sim = ctx.data();
    RNG &rng = sim.rng;
    PhysicsSystem::reset(ctx);

    const int32_t total = episodeBodies(sim);
    const int32_t num_dyn = total - kNumStatic;
    int32_t side = 1;
    while (side * side < num_dyn) side++;
    const float pen = 0.5f * kCell * (float)side;
    sim.pen = pen;
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
        const int32_t gx = i % side, gy = i / side;
        Vector3 pos;
        pos.x = -pen + kCell * ((float)gx + 0.5f);
        pos.x += 0.6f * (rng.sampleUniform() - 0.5f);
        pos.y = -pen + kCell * ((float)gy + 0.5f);
        pos.y += 0.6f * (rng.sampleUniform() - 0.5f);
        pos.z = 0.8f + 1.5f * rng.sampleUniform();
        Diag3x3 scale { 1.f, 1.f, 1.f };
        if (obj == SimObject::Ball) {
            const float s = 0.8f + 0.3f * rng.sampleUniform();
            scale = Diag3x3 { s, s, s };
        } else {
            scale.d0 = 0.5f + 0.4f * rng.sampleUniform();
            scale.d1 = 0.5f + 0.4f * rng.sampleUniform();
            scale.d2 = 0.5f + 0.4f * rng.sampleUniform();
        }
        Vector3 vel;
        vel.x = 6.f * (rng.sampleUniform() - 0.5f);
        vel.y = 6.f * (rng.sampleUniform() - 0.5f);
        vel.z = 0.f;
        const Quat rot = obj == SimObject::Ball ? upright : randomQuat(rng);
        sim.bodies[n++] = makeBody(ctx, pos, rot, scale, obj, ResponseType::Dynamic, vel);
    }
    sim.numBodies = n;
    ctx.singleton<BodyCount>().count = n;
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

static inline float signedUnit(RNG &rng)
{
    return 2.f * rng.sampleUniform() - 1.f;
}

// A point of the pen's air: within the walls, 0.1 to 4 m up
static inline Vector3 penPoint(RNG &rng, float pen)
{
    Vector3 p;
    p.x = pen * signedUnit(rng);
    p.y = pen * signedUnit(rng);
    p.z = 0.1f + 3.9f * rng.sampleUniform();
    return p;
}

static inline Vector3 randomDir(RNG &rng)
{
    Vector3 d;
    d.x = signedUnit(rng);
    d.y = signedUnit(rng);
    d.z = signedUnit(rng);
    return d;
}

// Before physics: this row's ray for the step, by row index (mod 8):
//   0, 1  towards a random body (unnormalised: t = 1 at its centre)
//   2     random origin and direction
//   3     along an axis; the other two components +0.f or -0.f
//   4     from a random dynamic body's centre (inside its hull)
//   5     parallel to the plane (d.z = 0)
//   6     from below the plane
//   7     towards a random body with max_t short of its centre (even steps) or +inf
inline void raySetupSystem(Engine &ctx, RayOrigin &origin, RayDir &dir, RayMaxT &max_t, RayState &st)
{
    const Sim &sim = ctx.data();
    RNG &rng = st.rng;
    const float inf = INFINITY;
    Vector3 o = penPoint(rng, sim.pen);
    Vector3 d = randomDir(rng);
    float t_max = inf;
    const int32_t kind = st.index % 8;
    if (kind == 0 || kind == 1 || kind == 7) {
        const int32_t b = rng.sampleI32(0, sim.numBodies);
        d = ctx.get<Position>(sim.bodies[b]) - o;
        if (kind == 7 && sim.stepInEpisode % 2 == 0) t_max = 0.5f * rng.sampleUniform();
    } else if (kind == 3) {
        const int32_t axis = rng.sampleI32(0, 3);
        const float sign = rng.sampleBool() ? 1.f : -1.f;
        const float z0 = rng.sampleBool() ? 0.f : -0.f;
        const float z1 = rng.sampleBool() ? 0.f : -0.f;
        if (axis == 0) d = Vector3 { sign, z0, z1 };
        else if (axis == 1) d = Vector3 { z0, sign, z1 };
        else d = Vector3 { z0, z1, sign };
    } else if (kind == 4 && sim.numBodies > kNumStatic) {
        const int32_t b = rng.sampleI32(kNumStatic, sim.numBodies);
        o = ctx.get<Position>(sim.bodies[b]);
    } else if (kind == 5) {
        d.z = 0.f;
    } else if (kind == 6) {
        o.z = -0.5f - rng.sampleUniform();
    }
    origin.v = o;
    dir.v = d;
    max_t.v = t_max;
}

// Last node: traceRay for the row's ray against the tree as the step left it
inline void rayProbeSystem(Engine &ctx, const RayOrigin &origin, const RayDir &dir, const RayMaxT &max_t,
                           HitEntity &hit, HitT &hit_t, HitNormal &hit_normal)
{
    float t = 0.f;
    Vector3 normal { 0, 0, 0 };
    const Entity e = ctx.singleton<broadphase::BVH>().traceRay(origin.v, dir.v, &t, &normal, max_t.v);
    hit.e = e;
    hit_t.v = e == Entity::none() ? 0.f : t;
    hit_normal.v = e == Entity::none() ? Vector3 { 0, 0, 0 } : normal;
}

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);
    auto setup = builder.addToGraph<ParallelForNode<Engine, raySetupSystem, RayOrigin, RayDir, RayMaxT,
                                                    RayState>>({});
    auto broadphase = PhysicsSystem::setupBroadphaseTasks(builder, {setup});
    auto physics = PhysicsSystem::setupPhysicsStepTasks(builder, {broadphase}, kNumSubsteps);
    auto cleanup = PhysicsSystem::setupCleanupTasks(builder, {physics});
    auto episode = builder.addToGraph<ParallelForNode<Engine, episodeSystem, BodyCount>>({cleanup});
    // destroyed bodies leave holes (CPU) / unsorted rows (GPU)
    auto compact = builder.addToGraph<CompactArchetypeNode<Body>>({episode});
#ifdef MADRONA_GPU_MODE
    auto post_reset = builder.addToGraph<RecycleEntitiesNode>({compact});
#else
    auto post_reset = compact;
#endif
    // a respawn re-registered every body: the broadphase rebuilds the tree
    auto post_bvh = PhysicsSystem::setupBroadphaseTasks(builder, {post_reset});
    builder.addToGraph<ParallelForNode<Engine, rayProbeSystem, RayOrigin, RayDir, RayMaxT, HitEntity, HitT,
                                       HitNormal>>({post_bvh});
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx),
      rng(init.seed),
      seed(init.seed),
      episodeLen(cfg.episodeLen),
      uniformBodies(cfg.uniformBodies),
      variedBodies(cfg.variedBodies != 0 ? cfg.variedBodies : (uint32_t)kVariedMaxBodies),
      stepInEpisode(0),
      episode(0),
      pen(0.f),
      numBodies(0)
{
    PhysicsSystem::init(ctx, cfg.objMgr, kDeltaT, kNumSubsteps, -9.8f * math::up,
                        cfg.uniformBodies != 0 ? (CountT)cfg.uniformBodies : (CountT)variedBodies);
    for (int32_t i = 0; i < kRaysPerWorld; i++) {
        Entity r = ctx.makeEntity<RayProbe>();
        ctx.get<RayOrigin>(r).v = Vector3::zero();
        ctx.get<RayDir>(r).v = Vector3::zero();
        ctx.get<RayMaxT>(r).v = 0.f;
        ctx.get<HitEntity>(r).e = Entity::none();
        ctx.get<HitT>(r).v = 0.f;
        ctx.get<HitNormal>(r).v = Vector3::zero();
        ctx.get<RayState>(r) = RayState { RNG(init.seed * (uint32_t)kRaysPerWorld + (uint32_t)i + 0x9e37u), i };
    }
    spawnWorld(ctx);
}

}

#ifdef MADRONA_GPU_MODE
MADRONA_BUILD_MWGPU_ENTRY(rays::Engine, rays::Sim, rays::Config, rays::WorldInit);
#endif
