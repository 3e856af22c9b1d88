#include "sim.hpp"

#ifdef MADRONA_GPU_MODE
#include <madrona/mw_gpu_entry.hpp>
#endif

using namespace madrona;
using namespace madrona::math;
using namespace madrona::phys;

namespace room {

constexpr float kDeltaT = 0.04f;
constexpr CountT kNumSubsteps = 4;
constexpr float kHalfWidth = 10.f;     // arena: x in [-10, 10]
constexpr float kLength = 30.f;        //        y in [0, 30]
constexpr float kWallThick = 0.5f;
constexpr float kWallHeight = 2.f;
constexpr float kDoorWidth = 3.f;
#ifdef ROOM_TGS
// build variant: the reference's TGS solver selected through the same API (its contact /
// joint solves are empty in the reference, src/physics/tgs.cpp: bodies fall freely)
constexpr PhysicsSystem::Solver kSolver = PhysicsSystem::Solver::TGS;
#else
constexpr PhysicsSystem::Solver kSolver = PhysicsSystem::Solver::XPBD;
#endif

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    base::registerTypes(registry);
    PhysicsSystem::registerTypes(registry, kSolver);
#ifdef ROOM_ENABLE_RENDER
    render::RenderingSystem::registerTypes(registry, nullptr);
#endif

    registry.registerComponent<Action>();
    registry.registerComponent<Reward>();
    registry.registerComponent<Done>();
    registry.registerComponent<Progress>();
    registry.registerComponent<StepsRemaining>();
    registry.registerComponent<SelfObs>();
    registry.registerComponent<Lidar>();
    registry.registerComponent<EntityType>();

    registry.registerSingleton<WorldReset>();
    registry.registerSingleton<BodyCount>();

    registry.registerArchetype<Agent>(
        ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumAgents);
    registry.registerArchetype<PhysicsEntity>();

    registry.exportSingleton<WorldReset>((uint32_t)ExportID::Reset);
    registry.exportColumn<Agent, Action>((uint32_t)ExportID::Action);
    registry.exportColumn<Agent, Reward>((uint32_t)ExportID::Reward);
    registry.exportColumn<Agent, Done>((uint32_t)ExportID::Done);
    registry.exportColumn<Agent, SelfObs>((uint32_t)ExportID::SelfObs);
    registry.exportColumn<Agent, Lidar>((uint32_t)ExportID::Lidar);
    registry.exportColumn<Agent, Position>((uint32_t)ExportID::AgentPos);
    registry.exportColumn<Agent, Rotation>((uint32_t)ExportID::AgentRot);
    registry.exportSingleton<BodyCount>((uint32_t)ExportID::BodyCount);
    registry.exportColumn<PhysicsEntity, Position>((uint32_t)ExportID::BodyPos);
    registry.exportColumn<PhysicsEntity, Rotation>((uint32_t)ExportID::BodyRot);
    registry.exportColumn<PhysicsEntity, Entity>((uint32_t)ExportID::BodyEntity);
    registry.exportColumn<PhysicsEntity, Velocity>((uint32_t)ExportID::BodyVel);
#ifdef ROOM_ENABLE_RENDER
    registry.exportColumn<render::RaycastOutputArchetype, render::RGBOutputBuffer>(
        (uint32_t)ExportID::RenderRGB);
    registry.exportColumn<render::RaycastOutputArchetype, render::DepthOutputBuffer>(
        (uint32_t)ExportID::RenderDepth);
    registry.exportColumn<PhysicsEntity, Scale>((uint32_t)ExportID::BodyScale);
    registry.exportColumn<PhysicsEntity, ObjectID>((uint32_t)ExportID::BodyObject);
    registry.exportColumn<Agent, Entity>((uint32_t)ExportID::AgentEntity);
    registry.exportColumn<render::RaycastOutputArchetype, render::SegmentationOutputBuffer>(
        (uint32_t)ExportID::RenderSegmentation);
#endif
}

static inline void setupBody(Engine &ctx, Entity e, Vector3 pos, Quat rot,
                             Diag3x3 scale, SimObject obj, ResponseType resp,
                             EntityType type)
{
    ObjectID obj_id { (int32_t)obj };
    ctx.get<Position>(e) = pos;
    ctx.get<Rotation>(e) = rot;
    ctx.get<Scale>(e) = scale;
    ctx.get<ObjectID>(e) = obj_id;
    ctx.get<ResponseType>(e) = resp;
    ctx.get<Velocity>(e) = Velocity { Vector3::zero(), Vector3::zero() };
    ctx.get<ExternalForce>(e) = Vector3::zero();
    ctx.get<ExternalTorque>(e) = Vector3::zero();
    ctx.get<EntityType>(e) = type;
    ctx.get<broadphase::LeafID>(e) = PhysicsSystem::registerEntity(ctx, e, obj_id);
#ifdef ROOM_ENABLE_RENDER
    render::RenderingSystem::makeEntityRenderable(ctx, e);
#endif
}

static inline void placeWall(Engine &ctx, Entity e, float x0, float x1,
                             float y0, float y1)
{
    Vector3 pos { 0.5f * (x0 + x1), 0.5f * (y0 + y1), 0.5f * kWallHeight };
    Diag3x3 scale { x1 - x0, y1 - y0, kWallHeight };
    setupBody(ctx, e, pos, Quat { 1, 0, 0, 0 }, scale, SimObject::Wall,
              ResponseType::Static, EntityType::Wall);
}

// (Re)generate the layout of this world.  Persistent entities (plane, walls,
// pillars, agents) are re-placed and re-registered with the broadphase; cubes
// are created fresh (the previous ones were destroyed by the caller).
static void generateWorld(Engine &ctx)
{
    Sim &sim = ctx.data();
    RNG &rng = sim.rng;

    PhysicsSystem::reset(ctx);

    setupBody(ctx, sim.plane, Vector3 { 0, 0, 0 }, Quat { 1, 0, 0, 0 },
              Diag3x3 { 1, 1, 1 }, SimObject::Plane, ResponseType::Static,
              EntityType::Plane);

    const float hw = kHalfWidth, t = kWallThick;
    placeWall(ctx, sim.borders[0], -hw - t, hw + t, -t, 0.f);
    placeWall(ctx, sim.borders[1], -hw - t, hw + t, kLength, kLength + t);
    placeWall(ctx, sim.borders[2], -hw - t, -hw, 0.f, kLength);
    placeWall(ctx, sim.borders[3], hw, hw + t, 0.f, kLength);

    // two interior walls, each with two door gaps -> three segments
    for (int32_t w = 0; w < 2; w++) {
        float y = (w == 0) ? 10.f : 20.f;
        float door_a = -hw + 1.f + rng.sampleUniform() * (hw - 2.f - kDoorWidth);
        float door_b = 1.f + rng.sampleUniform() * (hw - 2.f - kDoorWidth);
        placeWall(ctx, sim.inner[w * 3 + 0], -hw, door_a, y, y + t);
        placeWall(ctx, sim.inner[w * 3 + 1], door_a + kDoorWidth, door_b, y, y + t);
        placeWall(ctx, sim.inner[w * 3 + 2], door_b + kDoorWidth, hw, y, y + t);
    }

    for (int32_t i = 0; i < kNumPillars; i++) {
        float x = -8.f + 4.f * (float)i + (rng.sampleUniform() - 0.5f);
        float y = 4.f + 5.f * (float)i + (rng.sampleUniform() - 0.5f);
        setupBody(ctx, sim.pillars[i], Vector3 { x, y, 1.f }, Quat { 1, 0, 0, 0 },
                  Diag3x3 { 1.f, 1.f, 2.f }, SimObject::Wall, ResponseType::Static,
                  EntityType::Wall);
    }

    // cubes: one per cell of a 3 x 5 grid, jittered; some start in the air
    for (int32_t i = 0; i < kNumCubes; i++) {
        int32_t col = i % 3, row = i / 3;
        float x = -6.f + 6.f * (float)col + (rng.sampleUniform() - 0.5f) * 3.f;
        float y = 2.5f + 5.5f * (float)row + (rng.sampleUniform() - 0.5f) * 2.f;
        float z = 0.75f + (rng.sampleI32(0, 4) == 0 ? 1.5f : 0.f);
        Entity cube = ctx.makeEntity<PhysicsEntity>();
        sim.cubes[i] = cube;
        setupBody(ctx, cube, Vector3 { x, y, z }, Quat { 1, 0, 0, 0 },
                  Diag3x3 { 1.5f, 1.5f, 1.5f }, SimObject::Cube,
                  ResponseType::Dynamic, EntityType::Cube);
    }

    for (int32_t i = 0; i < kNumAgents; i++) {
        Entity agent = sim.agents[i];
        float x = (i == 0 ? -3.f : 3.f) + (rng.sampleUniform() - 0.5f);
        float y = 1.25f + rng.sampleUniform() * 0.5f;
        setupBody(ctx, agent, Vector3 { x, y, 0.75f }, Quat { 1, 0, 0, 0 },
                  Diag3x3 { 1.f, 1.f, 1.5f }, SimObject::Agent,
                  ResponseType::Dynamic, EntityType::Agent);
        ctx.get<Progress>(agent).maxY = y;
        ctx.get<StepsRemaining>(agent).t = sim.episodeLen;
    }
    sim.episode += 1;
}

// 45-degree steps: literal constants, no trigonometry at run time
static inline Vector3 moveDir(int32_t angle)
{
    constexpr float d = 0.70710678f;
    switch (angle & 7) {
    case 0: return Vector3 { 0, 1, 0 };
    case 1: return Vector3 { d, d, 0 };
    case 2: return Vector3 { 1, 0, 0 };
    case 3: return Vector3 { d, -d, 0 };
    case 4: return Vector3 { 0, -1, 0 };
    case 5: return Vector3 { -d, -d, 0 };
    case 6: return Vector3 { -1, 0, 0 };
    default: return Vector3 { -d, d, 0 };
    }
}

inline void movementSystem(Engine &, Action &action, Rotation &rot,
                           ExternalForce &force, ExternalTorque &torque)
{
    constexpr float move_max = 4000.f;
    constexpr float turn_max = 320.f;
    float f = move_max * (float)action.moveAmount * (1.f / 3.f);
    Vector3 dir = moveDir(action.moveAngle);
    Quat q = rot;
    force = q.rotateVec(Vector3 { f * dir.x, f * dir.y, 0.f });
    float t_z = turn_max * ((float)action.rotate - 2.f) * 0.5f;
    torque = Vector3 { 0.f, 0.f, t_z };
}

inline void agentZeroVelSystem(Engine &, Velocity &vel, Action &)
{
    vel.linear.x = 0.f;
    vel.linear.y = 0.f;
    vel.linear.z = fminf(vel.linear.z, 0.f);
    vel.angular = Vector3::zero();
}

inline void rewardSystem(Engine &, Position &pos, Progress &progress,
                         Reward &reward, StepsRemaining &steps, Done &done)
{
    float y = pos.y;
    float gain = 0.f;
    if (y > progress.maxY) {
        gain = (y - progress.maxY) * 0.05f;
        progress.maxY = y;
    }
    reward.v = gain;
    steps.t -= 1;
    done.v = steps.t == 0 ? 1 : 0;
}

inline void resetSystem(Engine &ctx, WorldReset &reset)
{
    Sim &sim = ctx.data();
    bool should_reset = reset.reset != 0;
    for (int32_t i = 0; i < kNumAgents; i++) {
        if (ctx.get<Done>(sim.agents[i]).v != 0) {
            should_reset = true;
        }
    }
    if (should_reset) {
        reset.reset = 0;
        if (sim.hasJoint != 0) {
            ctx.destroyEntity(sim.joint);
            sim.hasJoint = 0;
        }
        for (int32_t i = 0; i < kNumCubes; i++) {
            ctx.destroyEntity(sim.cubes[i]);
        }
        generateWorld(ctx);
    }
    ctx.singleton<BodyCount>().count =
        1 + kNumBorderWalls + kNumInnerWalls + kNumPillars + kNumCubes;
}

// One invocation per world.  Toggle a fixed joint between agent 0 and a cube.
inline void grabSystem(Engine &ctx, BodyCount &)
{
    Sim &sim = ctx.data();
    if (sim.grabPeriod == 0) {
        return;
    }
    sim.stepCount += 1;
    if (sim.stepCount % sim.grabPeriod != 0) {
        return;
    }
    if (sim.hasJoint != 0) {
        ctx.destroyEntity(sim.joint);
        sim.hasJoint = 0;
        return;
    }
    Entity agent = sim.agents[0];
    Vector3 agent_pos = ctx.get<Position>(agent);
    Quat agent_rot = ctx.get<Rotation>(agent);
    Vector3 hold_point = agent_pos + agent_rot.rotateVec(Vector3 { 0.f, 1.75f, 0.f });
    for (int32_t i = 0; i < kNumCubes; i++) {
        Vector3 cube_pos = ctx.get<Position>(sim.cubes[i]);
        if (cube_pos.distance2(hold_point) < 4.f) {
            sim.joint = PhysicsSystem::makeFixedJoint(ctx, agent, sim.cubes[i],
                Quat { 1, 0, 0, 0 }, Quat { 1, 0, 0, 0 },
                Vector3 { 0.f, 1.75f, 0.f }, Vector3 { 0.f, 0.f, 0.f }, 0.f);
            sim.hasJoint = 1;
            break;
        }
    }
}

inline void observationSystem(Engine &, Position &pos, Rotation &rot,
                              Progress &progress, StepsRemaining &steps,
                              SelfObs &obs)
{
    obs.x = pos.x * (1.f / kHalfWidth);
    obs.y = pos.y * (1.f / kLength);
    obs.z = pos.z;
    obs.qw = rot.w;
    obs.qx = rot.x;
    obs.qy = rot.y;
    obs.qz = rot.z;
    obs.maxY = progress.maxY * (1.f / kLength);
    obs.stepsRemaining = (float)steps.t;
}

inline void lidarSystem(Engine &ctx, Entity e, Position &pos, Rotation &rot,
                        Lidar &lidar)
{
    // unit directions at multiples of 22.5 degrees (literals)
    constexpr float c1 = 0.92387953f, s1 = 0.38268343f, d = 0.70710678f;
    const Vector3 dirs[kNumLidar] = {
        { 0, 1, 0 }, { s1, c1, 0 }, { d, d, 0 }, { c1, s1, 0 },
        { 1, 0, 0 }, { c1, -s1, 0 }, { d, -d, 0 }, { s1, -c1, 0 },
        { 0, -1, 0 }, { -s1, -c1, 0 }, { -d, -d, 0 }, { -c1, -s1, 0 },
        { -1, 0, 0 }, { -c1, s1, 0 }, { -d, d, 0 }, { -s1, c1, 0 },
    };
    broadphase::BVH &bvh = ctx.singleton<broadphase::BVH>();
    Quat q = rot;
    Vector3 origin = pos;
    origin.z += 0.25f;
#ifdef MADRONA_GPU_MODE
    // GPU backend: the node below runs kNumLidar threads per agent, one ray each
    // (same pattern as the upstream simulators' warp-level lidar)
    const int32_t first_ray = (int32_t)(threadIdx.x % kNumLidar);
    const int32_t last_ray = first_ray + 1;
#else
    const int32_t first_ray = 0;
    const int32_t last_ray = kNumLidar;
#endif
    for (int32_t i = first_ray; i < last_ray; i++) {
        Vector3 ray_dir = q.rotateVec(dirs[i]);
        // start just outside the agent's own (rotating) box
        Vector3 ray_o = origin + 0.8f * ray_dir;
        float hit_t;
        Vector3 hit_normal;
        Entity hit = bvh.traceRay(ray_o, ray_dir, &hit_t, &hit_normal, 200.f);
        if (hit == Entity::none() || hit == e) {
            lidar.samples[i] = LidarSample { 0.f, 0.f };
        } else {
            EntityType type = ctx.get<EntityType>(hit);
            lidar.samples[i] = LidarSample { hit_t, (float)(uint32_t)type };
        }
    }
}

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);

    auto move = builder.addToGraph<ParallelForNode<Engine, movementSystem,
        Action, Rotation, ExternalForce, ExternalTorque>>({});

    auto broadphase = PhysicsSystem::setupBroadphaseTasks(builder, {move});
    auto physics = PhysicsSystem::setupPhysicsStepTasks(builder, {broadphase},
                                                        kNumSubsteps, kSolver);

    auto zero_vel = builder.addToGraph<ParallelForNode<Engine, agentZeroVelSystem,
        Velocity, Action>>({physics});
    auto cleanup = PhysicsSystem::setupCleanupTasks(builder, {zero_vel});

    auto grab = builder.addToGraph<ParallelForNode<Engine, grabSystem,
        BodyCount>>({cleanup});
    auto reward = builder.addToGraph<ParallelForNode<Engine, rewardSystem,
        Position, Progress, Reward, StepsRemaining, Done>>({grab});
    auto reset = builder.addToGraph<ParallelForNode<Engine, resetSystem,
        WorldReset>>({reward});

    // destroyed cubes leave holes (CPU) / unsorted rows (GPU)
    auto compact = builder.addToGraph<CompactArchetypeNode<PhysicsEntity>>({reset});
#ifdef MADRONA_GPU_MODE
    auto recycle = builder.addToGraph<RecycleEntitiesNode>({compact});
    auto post_reset = recycle;
#else
    auto post_reset = compact;
#endif
    // a reset re-registered every body: rebuild the tree so lidar sees the new world
    auto post_bvh = PhysicsSystem::setupBroadphaseTasks(builder, {post_reset});

    auto obs = builder.addToGraph<ParallelForNode<Engine, observationSystem,
        Position, Rotation, Progress, StepsRemaining, SelfObs>>({post_bvh});
    // independent of the observation system: a parallel branch of the step graph on the GPU
#ifdef MADRONA_GPU_MODE
    builder.addToGraph<CustomParallelForNode<Engine, lidarSystem, kNumLidar, 1,
        Entity, Position, Rotation, Lidar>>({post_bvh});
#else
    builder.addToGraph<ParallelForNode<Engine, lidarSystem,
        Entity, Position, Rotation, Lidar>>({post_bvh});
#endif
#ifdef ROOM_ENABLE_RENDER
    render::RenderingSystem::setupTasks(builder, {obs});
#endif
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx),
      rng(init.seed),
      episodeLen(cfg.episodeLen),
      episode(0),
      grabPeriod(cfg.grabPeriod),
      stepCount(0),
      hasJoint(0),
      joint(Entity::none())
{
    PhysicsSystem::init(ctx, cfg.objMgr, kDeltaT, kNumSubsteps,
                        -9.8f * math::up, kMaxBodies, kSolver);

    plane = ctx.makeEntity<PhysicsEntity>();
    for (int32_t i = 0; i < kNumBorderWalls; i++) {
        borders[i] = ctx.makeEntity<PhysicsEntity>();
    }
    for (int32_t i = 0; i < kNumInnerWalls; i++) {
        inner[i] = ctx.makeEntity<PhysicsEntity>();
    }
    for (int32_t i = 0; i < kNumPillars; i++) {
        pillars[i] = ctx.makeEntity<PhysicsEntity>();
    }
    for (int32_t i = 0; i < kNumAgents; i++) {
        agents[i] = ctx.makeEntity<Agent>();
        ctx.get<Action>(agents[i]) = Action { 0, 0, 2 };
        ctx.get<Done>(agents[i]).v = 0;
        ctx.get<Reward>(agents[i]).v = 0.f;
        ctx.get<SelfObs>(agents[i]) = SelfObs {};
        ctx.get<Lidar>(agents[i]) = Lidar {};
#ifdef ROOM_ENABLE_RENDER
        render::RenderingSystem::attachEntityToView(ctx, agents[i], 90.f, 0.001f,
                                                   Vector3 { 0.f, 0.f, 0.5f });
#endif
    }
    ctx.singleton<WorldReset>().reset = 0;
    generateWorld(ctx);
    ctx.singleton<BodyCount>().count =
        1 + kNumBorderWalls + kNumInnerWalls + kNumPillars + kNumCubes;
}

}

#ifdef MADRONA_GPU_MODE
MADRONA_BUILD_MWGPU_ENTRY(room::Engine, room::Sim, room::Config, room::WorldInit);
#endif
