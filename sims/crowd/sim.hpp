// Fixture simulator "crowd": a walled pen (plane and four static walls) filled with boxes,
// spheres, wedges and pentagonal pyramids thrown about, so that hull - hull, sphere - hull,
// sphere - sphere, sphere - plane and hull - plane pairs all occur.  A world's body count
// (plane and walls included) comes from its seed and episode number, from
// kEpisodeSizes, on both sides of the engine's 128-body warp-per-world path; every
// episode_len steps the world destroys its bodies, resets the broadphase and respawns with
// the next size, so worlds cross 128 bodies in both directions and the tree is rebuilt at
// every size.  Config::uniformBodies > 0 gives every world and episode that count instead.
//
// Bodies are spread over a pen that grows with the count (one 2 m cell each), so the trees
// stay as shallow as a uniform spread makes them and within the reference's own 32-entry
// query stacks (include/madrona/broadphase.inl:24).  Layout::Clustered instead packs the
// bodies towards one corner in a geometric spiral, a tree deeper than the rebuild's
// 64-entry stacks: the engine must refuse it (GPU only).
//
// Compiled unchanged for the reference CPU backend (oracle/harness_crowd.cpp) and,
// through NVRTC, for this engine.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/components.hpp>
#include <madrona/physics.hpp>
#include <madrona/rand.hpp>

namespace crowd {

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

constexpr int32_t kNumStatic = 5;          // plane and four walls
constexpr int32_t kMaxBodies = 4096;       // per world, static bodies included
constexpr int32_t kVariedMaxBodies = 1500; // the largest of kEpisodeSizes
constexpr int32_t kNumEpisodeSizes = 7;

enum class ExportID : uint32_t {
    BodyPos,
    BodyRot,
    BodyVel,
    BodyEntity,
    BodyCount,
    NumExports,
};

enum class TaskGraphID : uint32_t {
    Step,
    NumTaskGraphs,
};

// indices into the ObjectManager built by sims/objects.py:hullpile_objects()
enum class SimObject : uint32_t {
    Box,
    Wedge,
    OctPrism,
    Bipyramid,
    Tetra,
    PentaPyramid,
    Ball,
    Dumbbell,
    CappedBox,
    Plane,
    Wall,
    Pedestal,
    NumObjects,
};

// Config::layout
enum class Layout : uint32_t {
    Spread,            // the fixture
    Clustered,         // a geometric spiral: a tree too deep for the rebuild's stacks
};

struct BodyCount {
    int32_t count;
};

struct Body : public madrona::Archetype<madrona::phys::RigidBody> {};

struct Config {
    madrona::phys::ObjectManager *objMgr;
    uint32_t episodeLen;
    uint32_t uniformBodies;    // 0: the sizes of kEpisodeSizes
    uint32_t layout;
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
    uint32_t seed;
    uint32_t episodeLen;
    uint32_t uniformBodies;
    uint32_t layout;
    uint32_t stepInEpisode;
    uint32_t episode;
    int32_t numBodies;
    Entity bodies[kMaxBodies];
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
