// Fixture simulator 3 ("rigid-body room", BASELINE.json configs[1]: the
// Escape-Room-class workload).  Per world: a ground plane, border and interior
// walls with door gaps, static pillars, pushable cubes and two force-driven
// agents = 33 rigid bodies; XPBD with 4 substeps at dt = 0.04; 16-ray lidar
// through the broadphase tree; cubes are destroyed and recreated on every
// episode reset (entity churn + compaction).  The upstream Escape Room sources
// are not available here (SURVEY.md F7); this fixture defines the workload by
// construction.  No transcendental functions: directions come from literal
// tables, so with FP contraction off on both sides floats can be compared
// tightly against the reference CPU backend.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/components.hpp>
#include <madrona/physics.hpp>
#include <madrona/rand.hpp>
#ifdef ROOM_ENABLE_RENDER
// GPU-only build variant (BASELINE.json configs[3]): every body is renderable,
// every agent carries a camera; the batch ray caster writes depth / RGB.
#include <madrona/render/ecs.hpp>
#endif

namespace room {

using madrona::Entity;
using madrona::CountT;
using madrona::base::Position;
using madrona::base::Rotation;
using madrona::base::Scale;
using madrona::base::ObjectID;
using madrona::phys::Velocity;
using madrona::phys::ResponseType;
using madrona::phys::ExternalForce;
using madrona::phys::ExternalTorque;

constexpr int32_t kNumAgents = 2;
constexpr int32_t kNumCubes = 15;
constexpr int32_t kNumBorderWalls = 4;
constexpr int32_t kNumInnerWalls = 6;
constexpr int32_t kNumPillars = 5;
constexpr int32_t kNumLidar = 16;
constexpr int32_t kMaxBodies = 40;

enum class ExportID : uint32_t {
    Reset,
    Action,
    Reward,
    Done,
    SelfObs,
    Lidar,
    AgentPos,
    AgentRot,
    BodyCount,
    BodyPos,
    BodyRot,
    BodyEntity,
    BodyVel,
#ifdef ROOM_ENABLE_RENDER
    RenderRGB,
    RenderDepth,
    BodyScale,
    BodyObject,
    AgentEntity,
    RenderSegmentation,
#endif
    NumExports,
};

enum class TaskGraphID : uint32_t {
    Step,
    NumTaskGraphs,
};

enum class SimObject : uint32_t {
    Cube,
    Wall,
    Agent,
    Plane,
    NumObjects,
};

enum class EntityType : uint32_t {
    None,
    Cube,
    Wall,
    Agent,
    Plane,
};

struct WorldReset { int32_t reset; };
struct BodyCount { int32_t count; };

struct Action {
    int32_t moveAmount;   // [0, 3]
    int32_t moveAngle;    // [0, 7], multiples of 45 degrees in the agent frame
    int32_t rotate;       // [0, 4], 2 = none
};

struct Reward { float v; };
struct Done { int32_t v; };

struct Progress { float maxY; };
struct StepsRemaining { uint32_t t; };

struct SelfObs {
    float x, y, z;
    float qw, qx, qy, qz;
    float maxY;
    float stepsRemaining;
};

struct LidarSample {
    float depth;
    float type;
};

struct Lidar {
    LidarSample samples[kNumLidar];
};

#ifdef ROOM_ENABLE_RENDER
struct Agent : public madrona::Archetype<
    madrona::phys::RigidBody,
    Action, Reward, Done, Progress, StepsRemaining, SelfObs, Lidar, EntityType,
    madrona::render::Renderable, madrona::render::RenderCamera
> {};

struct PhysicsEntity : public madrona::Archetype<
    madrona::phys::RigidBody,
    EntityType,
    madrona::render::Renderable
> {};
#else
struct Agent : public madrona::Archetype<
    madrona::phys::RigidBody,
    Action, Reward, Done, Progress, StepsRemaining, SelfObs, Lidar, EntityType
> {};

struct PhysicsEntity : public madrona::Archetype<
    madrona::phys::RigidBody,
    EntityType
> {};
#endif

struct Config {
    madrona::phys::ObjectManager *objMgr;
    uint32_t episodeLen;
    // > 0: every grabPeriod steps agent 0 grabs the next cube in reach with a
    // fixed joint, or lets go of the one it holds (exercises JointConstraint)
    uint32_t grabPeriod;
};

struct WorldInit {
    uint32_t seed;
};

class Engine;

struct Sim : public madrona::WorldBase {
    static void registerTypes(madrona::ECSRegistry &registry, const Config &cfg);
    static void setupTasks(madrona::TaskGraphManager &mgr, const Config &cfg);

    Sim(Engine &ctx, const Config &cfg, const WorldInit &init);

    madrona::RNG rng;
    uint32_t episodeLen;
    uint32_t episode;

    Entity plane;
    Entity borders[kNumBorderWalls];
    Entity inner[kNumInnerWalls];
    Entity pillars[kNumPillars];
    Entity cubes[kNumCubes];
    Entity agents[kNumAgents];

    uint32_t grabPeriod;
    uint32_t stepCount;
    uint32_t hasJoint;
    Entity joint;
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
