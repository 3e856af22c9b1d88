// Fixture simulator "buttons": Escape-Room-style pressure plates on top of the
// XPBD step.  Per world: a floor plane and four walls, two force-driven agents,
// loose cubes, a ball (sphere primitive) that starts on button 1, two buttons
// (plain entities outside the broadphase tree) and two doors (static bodies) that
// sink while their button is pressed and rise again when it is released.  After
// setupPhysicsStepTasks -- on a tree that was only refitted -- a per-button system
// asks findEntitiesWithinAABB what stands on the button, and a per-world system
// tests the agents against a goal zone with checkEntityAABBOverlap.  Episodes
// reset with PhysicsSystem::reset and re-registration, as in sims/arena.
// Compiled unchanged for the reference CPU backend (oracle/harness_buttons.cpp)
// and, through NVRTC, for this engine.  No transcendental functions.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/components.hpp>
#include <madrona/physics.hpp>
#include <madrona/rand.hpp>

namespace buttons {

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
constexpr int32_t kNumWalls = 4;
constexpr int32_t kNumCubes = 4;
constexpr int32_t kNumButtons = 2;
constexpr int32_t kNumDoors = kNumButtons;
// plane + walls + cubes + ball (the PhysicsEntity table)
constexpr int32_t kNumPhysicsEntities = 1 + kNumWalls + kNumCubes + 1;
constexpr int32_t kMaxBodies = kNumPhysicsEntities + kNumAgents + kNumDoors;

enum class ExportID : uint32_t {
    Reset,
    Action,
    ButtonState,
    DoorPos,
    AgentPos,
    Goal,
    BodyPos,
    BodyEntity,
    NumExports,
};

enum class TaskGraphID : uint32_t {
    Step,
    NumTaskGraphs,
};

// indices into the ObjectManager built by sims/objects.py:balls_objects()
enum class SimObject : uint32_t {
    Cube,
    Wall,
    Agent,
    Plane,
    Ball,
    NumObjects,
};

struct WorldReset { int32_t reset; };

struct Action {
    int32_t moveAmount;   // [0, 3]
    int32_t moveAngle;    // [0, 7], multiples of 45 degrees
    int32_t rotate;       // [0, 4], 2 = none
};

struct StepsRemaining { uint32_t t; };

// the agent overlaps the goal zone (checkEntityAABBOverlap)
struct InGoal { int32_t v; };

struct ButtonState {
    int32_t pressed;
    int32_t numFound;     // entities findEntitiesWithinAABB reported
    int32_t firstFound;   // entity id of the first report (-1: none)
    int32_t ballOn;       // the ball's centre is above the plate (the ball is never reported)
};

struct Agent : public madrona::Archetype<
    madrona::phys::RigidBody, Action, StepsRemaining, InGoal
> {};

struct PhysicsEntity : public madrona::Archetype<
    madrona::phys::RigidBody
> {};

struct Door : public madrona::Archetype<
    madrona::phys::RigidBody
> {};

// outside the broadphase tree: a position and what stands on it
struct Button : public madrona::Archetype<
    Position, ButtonState
> {};

struct Config {
    madrona::phys::ObjectManager *objMgr;
    uint32_t episodeLen;
    uint32_t pad;
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
    Entity plane;
    Entity walls[kNumWalls];
    Entity agents[kNumAgents];
    Entity doors[kNumDoors];
    Entity buttons[kNumButtons];
    // recreated on every episode reset
    Entity cubes[kNumCubes];
    Entity ball;
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
