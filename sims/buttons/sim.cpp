#include "sim.hpp"

#ifdef MADRONA_GPU_MODE
#include <madrona/mw_gpu_entry.hpp>
#endif

using namespace madrona;
using namespace madrona::math;
using namespace madrona::phys;

namespace buttons {

constexpr float kDeltaT = 0.04f;
constexpr CountT kNumSubsteps = 4;
constexpr float kHalf = 6.f;           // pen interior: [-6, 6]^2
constexpr float kWallThick = 0.5f;
constexpr float kWallHeight = 2.f;
constexpr float kBallScale = 1.2f;     // radius 0.6
constexpr float kButtonHalf = 0.7f;    // button plate: 1.4 x 1.4, 0.3 high
constexpr float kButtonHeight = 0.3f;
constexpr float kDoorUp = 1.f;         // door centre height when closed
constexpr float kDoorDown = -1.1f;     // fully sunk into the floor
constexpr float kDoorSpeed = 0.15f;    // per step

static inline AABB goalBox()
{
    return AABB { Vector3 { 1.5f, -2.5f, 0.f }, Vector3 { 6.f, 1.f, 2.f } };
}

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    base::registerTypes(registry);
    PhysicsSystem::registerTypes(registry);

    registry.registerComponent<Action>();
    registry.registerComponent<StepsRemaining>();
    registry.registerComponent<InGoal>();
    registry.registerComponent<ButtonState>();

    registry.registerSingleton<WorldReset>();

    registry.registerArchetype<Agent>(
        ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumAgents);
    registry.registerArchetype<PhysicsEntity>();
    registry.registerArchetype<Door>(
        ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumDoors);
    registry.registerArchetype<Button>(
        ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumButtons);

    registry.exportSingleton<WorldReset>((uint32_t)ExportID::Reset);
    registry.exportColumn<Agent, Action>((uint32_t)ExportID::Action);
    registry.exportColumn<Button, ButtonState>((uint32_t)ExportID::ButtonState);
    registry.exportColumn<Door, Position>((uint32_t)ExportID::DoorPos);
    registry.exportColumn<Agent, Position>((uint32_t)ExportID::AgentPos);
    registry.exportColumn<Agent, InGoal>((uint32_t)ExportID::Goal);
    registry.exportColumn<PhysicsEntity, Position>((uint32_t)ExportID::BodyPos);
    registry.exportColumn<PhysicsEntity, Entity>((uint32_t)ExportID::BodyEntity);
}

static inline void setupBody(Engine &ctx, Entity e, Vector3 pos, Diag3x3 scale,
                             SimObject obj, ResponseType resp)
{
    ObjectID obj_id { (int32_t)obj };
    ctx.get<Position>(e) = pos;
    ctx.get<Rotation>(e) = Quat { 1, 0, 0, 0 };
    ctx.get<Scale>(e) = scale;
    ctx.get<ObjectID>(e) = obj_id;
    ctx.get<ResponseType>(e) = resp;
    ctx.get<Velocity>(e) = Velocity { Vector3::zero(), Vector3::zero() };
    ctx.get<ExternalForce>(e) = Vector3::zero();
    ctx.get<ExternalTorque>(e) = Vector3::zero();
    ctx.get<broadphase::LeafID>(e) = PhysicsSystem::registerEntity(ctx, e, obj_id);
}

static inline float jitter(RNG &rng, float span)
{
    return (rng.sampleUniform() - 0.5f) * span;
}

// (Re)generate the layout of this world.  Persistent entities are re-placed and
// re-registered with the broadphase; cubes and the ball are created fresh (the
// previous ones were destroyed by the caller).
static void generateWorld(Engine &ctx)
{
    Sim &sim = ctx.data();
    RNG &rng = sim.rng;

    PhysicsSystem::reset(ctx);

    setupBody(ctx, sim.plane, Vector3 { 0, 0, 0 }, Diag3x3 { 1, 1, 1 }, SimObject::Plane,
              ResponseType::Static);
    const float reach = kHalf + kWallThick, mid = kHalf + 0.5f * kWallThick;
    const float hz = 0.5f * kWallHeight;
    setupBody(ctx, sim.walls[0], Vector3 { 0, -mid, hz }, Diag3x3 { 2.f * reach, kWallThick, kWallHeight },
              SimObject::Wall, ResponseType::Static);
    setupBody(ctx, sim.walls[1], Vector3 { 0, mid, hz }, Diag3x3 { 2.f * reach, kWallThick, kWallHeight },
              SimObject::Wall, ResponseType::Static);
    setupBody(ctx, sim.walls[2], Vector3 { -mid, 0, hz }, Diag3x3 { kWallThick, 2.f * kHalf, kWallHeight },
              SimObject::Wall, ResponseType::Static);
    setupBody(ctx, sim.walls[3], Vector3 { mid, 0, hz }, Diag3x3 { kWallThick, 2.f * kHalf, kWallHeight },
              SimObject::Wall, ResponseType::Static);

    for (int32_t i = 0; i < kNumAgents; i++) {
        const float x = (i == 0 ? -2.f : 2.f) + jitter(rng, 1.f);
        const float y = -3.5f + jitter(rng, 1.f);
        setupBody(ctx, sim.agents[i], Vector3 { x, y, 0.75f }, Diag3x3 { 1.f, 1.f, 1.5f },
                  SimObject::Agent, ResponseType::Dynamic);
        ctx.get<StepsRemaining>(sim.agents[i]).t = sim.episodeLen;
        ctx.get<InGoal>(sim.agents[i]).v = 0;
    }

    // button 0 in the agents' half, button 1 under the ball
    const Vector3 b0 { jitter(rng, 4.f), -1.f + jitter(rng, 2.f), 0.f };
    const Vector3 b1 { -3.5f + jitter(rng, 1.f), 2.f + jitter(rng, 1.f), 0.f };
    ctx.get<Position>(sim.buttons[0]) = b0;
    ctx.get<Position>(sim.buttons[1]) = b1;
    for (int32_t i = 0; i < kNumButtons; i++) {
        ctx.get<ButtonState>(sim.buttons[i]) = ButtonState { 0, 0, -1, 0 };
    }

    for (int32_t i = 0; i < kNumDoors; i++) {
        setupBody(ctx, sim.doors[i], Vector3 { i == 0 ? -1.5f : 1.5f, 4.5f, kDoorUp },
                  Diag3x3 { 2.f, 0.4f, 2.f }, SimObject::Wall, ResponseType::Static);
    }

    for (int32_t i = 0; i < kNumCubes; i++) {
        Entity cube = ctx.makeEntity<PhysicsEntity>();
        sim.cubes[i] = cube;
        const float x = -4.5f + 3.f * (float)i + jitter(rng, 1.f);
        const float y = jitter(rng, 6.f);
        setupBody(ctx, cube, Vector3 { x, y, 0.5f + (rng.sampleI32(0, 3) == 0 ? 1.f : 0.f) },
                  Diag3x3 { 1.f, 1.f, 1.f }, SimObject::Cube, ResponseType::Dynamic);
    }
    sim.ball = ctx.makeEntity<PhysicsEntity>();
    setupBody(ctx, sim.ball, Vector3 { b1.x, b1.y, 0.5f * kBallScale }, Diag3x3 { kBallScale, kBallScale, kBallScale },
              SimObject::Ball, ResponseType::Dynamic);
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
    const float f = move_max * (float)action.moveAmount * (1.f / 3.f);
    const Vector3 dir = moveDir(action.moveAngle);
    const Quat q = rot;
    force = q.rotateVec(Vector3 { f * dir.x, f * dir.y, 0.f });
    torque = Vector3 { 0.f, 0.f, turn_max * ((float)action.rotate - 2.f) * 0.5f };
}

inline void agentZeroVelSystem(Engine &, Velocity &vel, Action &)
{
    vel.linear.x = 0.f;
    vel.linear.y = 0.f;
    vel.linear.z = fminf(vel.linear.z, 0.f);
    vel.angular = Vector3::zero();
}

// what stands on the button: a query of the tree the physics step refitted
inline void buttonSystem(Engine &ctx, Position &pos, ButtonState &state)
{
    const AABB box { Vector3 { pos.x - kButtonHalf, pos.y - kButtonHalf, pos.z },
                     Vector3 { pos.x + kButtonHalf, pos.y + kButtonHalf, pos.z + kButtonHeight } };
    state.numFound = 0;
    state.firstFound = -1;
    PhysicsSystem::findEntitiesWithinAABB(ctx, box, [&](Entity e) {
        if (state.numFound == 0) state.firstFound = e.id;
        state.numFound += 1;
    });
    state.pressed = state.numFound > 0 ? 1 : 0;
    const Vector3 ball = ctx.get<Position>(ctx.data().ball);
    state.ballOn = (ball.x > box.pMin.x && ball.x < box.pMax.x &&
                    ball.y > box.pMin.y && ball.y < box.pMax.y) ? 1 : 0;
}

// doors follow their buttons, agents are tested against the goal zone, episodes reset
inline void worldSystem(Engine &ctx, WorldReset &reset)
{
    Sim &sim = ctx.data();
    for (int32_t i = 0; i < kNumDoors; i++) {
        Position &door = ctx.get<Position>(sim.doors[i]);
        if (ctx.get<ButtonState>(sim.buttons[i]).pressed != 0) {
            door.z = fmaxf(door.z - kDoorSpeed, kDoorDown);
        } else {
            door.z = fminf(door.z + kDoorSpeed, kDoorUp);
        }
    }

    bool should_reset = reset.reset != 0;
    for (int32_t i = 0; i < kNumAgents; i++) {
        ctx.get<InGoal>(sim.agents[i]).v =
            PhysicsSystem::checkEntityAABBOverlap(ctx, goalBox(), sim.agents[i]) ? 1 : 0;
        StepsRemaining &steps = ctx.get<StepsRemaining>(sim.agents[i]);
        steps.t -= 1;
        if (steps.t == 0) should_reset = true;
    }
    if (should_reset) {
        reset.reset = 0;
        for (int32_t i = 0; i < kNumCubes; i++) ctx.destroyEntity(sim.cubes[i]);
        ctx.destroyEntity(sim.ball);
        generateWorld(ctx);
    }
}

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);

    auto move = builder.addToGraph<ParallelForNode<Engine, movementSystem,
        Action, Rotation, ExternalForce, ExternalTorque>>({});
    auto broadphase = PhysicsSystem::setupBroadphaseTasks(builder, {move});
    auto physics = PhysicsSystem::setupPhysicsStepTasks(builder, {broadphase},
                                                        kNumSubsteps);
    auto zero_vel = builder.addToGraph<ParallelForNode<Engine, agentZeroVelSystem,
        Velocity, Action>>({physics});
    auto cleanup = PhysicsSystem::setupCleanupTasks(builder, {zero_vel});

    auto press = builder.addToGraph<ParallelForNode<Engine, buttonSystem,
        Position, ButtonState>>({cleanup});
    auto world = builder.addToGraph<ParallelForNode<Engine, worldSystem,
        WorldReset>>({press});

    auto compact = builder.addToGraph<CompactArchetypeNode<PhysicsEntity>>({world});
#ifdef MADRONA_GPU_MODE
    builder.addToGraph<RecycleEntitiesNode>({compact});
#else
    (void)compact;
#endif
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx),
      rng(init.seed),
      episodeLen(cfg.episodeLen)
{
    PhysicsSystem::init(ctx, cfg.objMgr, kDeltaT, kNumSubsteps,
                        -9.8f * math::up, kMaxBodies);

    plane = ctx.makeEntity<PhysicsEntity>();
    for (int32_t i = 0; i < kNumWalls; i++) walls[i] = ctx.makeEntity<PhysicsEntity>();
    for (int32_t i = 0; i < kNumAgents; i++) {
        agents[i] = ctx.makeEntity<Agent>();
        ctx.get<Action>(agents[i]) = Action { 0, 0, 2 };
    }
    for (int32_t i = 0; i < kNumDoors; i++) doors[i] = ctx.makeEntity<Door>();
    for (int32_t i = 0; i < kNumButtons; i++) buttons[i] = ctx.makeEntity<Button>();
    ctx.singleton<WorldReset>().reset = 0;
    generateWorld(ctx);
}

}

#ifdef MADRONA_GPU_MODE
MADRONA_BUILD_MWGPU_ENTRY(buttons::Engine, buttons::Sim, buttons::Config, buttons::WorldInit);
#endif
