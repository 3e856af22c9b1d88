// Fixture simulator "triggers": trigger volumes on the broadphase alone, no
// solver.  Per world: a floor plane, four static walls, two kinematic agents
// moved by actions, a kinematic compound "dumbbell" (two box hulls) and a
// kinematic ball (sphere) on fixed paths, and static pickups.  The step graph
// is: moves -> setupBroadphaseTasks -> setupStandaloneBroadphaseOverlapTasks ->
// user systems on the CandidateCollision rows -> cleanup.  A per-row system
// marks pickups that an agent or the dumbbell overlaps; a per-world system
// exports the world's first pairs, queries a zone with findEntitiesWithinAABB /
// checkEntityAABBOverlap, and replaces the marked pickups (destroy, create,
// PhysicsSystem::reset and re-registration).  Compiled unchanged for the
// reference CPU backend and, through NVRTC, for this engine.  No
// transcendental functions: paths and yaw angles come from literal tables.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/components.hpp>
#include <madrona/physics.hpp>
#include <madrona/rand.hpp>

namespace triggers {

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
using madrona::phys::CandidateCollision;

constexpr int32_t kNumAgents = 2;
constexpr int32_t kNumWalls = 4;
constexpr int32_t kNumPickups = 6;
constexpr int32_t kNumProps = 1 + kNumWalls + 2;        // floor, walls, dumbbell, ball
constexpr int32_t kMaxBodies = kNumProps + kNumAgents + kNumPickups;
constexpr int32_t kMaxPairs = 32;                        // pairs exported per world

enum class ExportID : uint32_t {
    Action,
    Pairs,
    Zone,
    AgentPos,
    PickupEntity,
    PickupPos,
    PropEntity,
    NumExports,
};

enum class TaskGraphID : uint32_t {
    Step,
    NumTaskGraphs,
};

// indices into the ObjectManager built by sims/objects.py:triggers_objects()
enum class SimObject : uint32_t {
    Agent,
    Pickup,
    Wall,
    Floor,
    Dumbbell,       // two box hulls
    Ball,           // one sphere
    NumObjects,
};

enum class Kind : uint32_t {
    Floor,
    Wall,
    Agent,
    Dumbbell,
    Ball,
    Pickup,
};

struct Action {
    int32_t dx;     // [0, 2], 1 = stay
    int32_t dy;
};

struct Touched { int32_t v; };

// the world's CandidateCollision rows, in the order ctx.iterateQuery reports them
struct PairObs {
    int32_t count;
    int32_t pairs[kMaxPairs][4];     // entity a id, entity b id, aPrim, bPrim
};

struct ZoneObs {
    int32_t numFound;       // findEntitiesWithinAABB reports
    int32_t firstFound;     // entity id of the first report (-1: none)
    int32_t agentInZone;    // checkEntityAABBOverlap(agent 0)
    int32_t dumbbellInZone; // checkEntityAABBOverlap(dumbbell)
    int32_t ballInZone;     // checkEntityAABBOverlap(ball): sphere only, never true
    int32_t ballCentreInZone;
    int32_t respawns;       // pickups replaced so far
    int32_t step;
};

struct Agent : public madrona::Archetype<
    madrona::phys::RigidBody, Kind, Action
> {};

struct Prop : public madrona::Archetype<
    madrona::phys::RigidBody, Kind
> {};

struct Pickup : public madrona::Archetype<
    madrona::phys::RigidBody, Kind, Touched
> {};

struct Config {
    madrona::phys::ObjectManager *objMgr;
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
    int32_t step;
    Entity floor;
    Entity walls[kNumWalls];
    Entity agents[kNumAgents];
    Entity dumbbell;
    Entity ball;
    Entity pickups[kNumPickups];
    madrona::Query<CandidateCollision> candQuery;
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
