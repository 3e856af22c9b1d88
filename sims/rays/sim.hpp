// Fixture simulator "rays": broadphase::BVH::traceRay probed from inside the simulator, to
// check the engine's batched physics ray queries (mb2_trace_physics_rays) against it.
//
// A walled pen (plane and four static walls) of boxes, wedges, octagonal prisms, pentagonal
// pyramids and two-box dumbbells (a two-hull compound), scaled and rotated, thrown about so
// they fall and collide and the trees are refit; every episode_len steps the world destroys its
// bodies and respawns, so the trees are rebuilt.  A world's body count comes from its seed and
// episode (8 to Config::variedBodies, so one batch can hold worlds on both sides of 128 leaves),
// or is Config::uniformBodies for every world.  Built with -DRAYS_SPHERES=1, every
// other ball-sized slot is a sphere (traceRay skips spheres; GPU only).
//
// Each world has kRaysPerWorld RayProbe rows.  raySetupSystem, the graph's first node, fills
// each row's ray from the row's own RNG (so both backends draw the same bits): rays aimed at
// bodies, random rays, axis-aligned directions with -0.f components, rays from inside hulls,
// rays parallel to the plane and from below it, max_t short of a hit or +inf.  rayProbeSystem,
// the graph's last node, calls traceRay for every row and stores the hit (entity, t, normal; a
// miss as Entity::none(), 0, 0).  Every column is exported in place.
//
// Compiled unchanged for the reference CPU backend and, through NVRTC, for this engine.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/components.hpp>
#include <madrona/physics.hpp>
#include <madrona/rand.hpp>

namespace rays {

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
constexpr int32_t kVariedMaxBodies = 60;   // Config::variedBodies = 0
constexpr int32_t kRaysPerWorld = 64;

enum class ExportID : uint32_t {
    RayOrigin,
    RayDir,
    RayMaxT,
    HitEntity,
    HitT,
    HitNormal,
    BodyCount,
    BodyPos,
    BodyEntity,
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

struct RayOrigin { madrona::math::Vector3 v; };
struct RayDir { madrona::math::Vector3 v; };
struct RayMaxT { float v; };
struct HitEntity { Entity e; };
struct HitT { float v; };
struct HitNormal { madrona::math::Vector3 v; };
struct RayState {
    madrona::RNG rng;
    int32_t index;             // row within the world
};

struct BodyCount {
    int32_t count;
};

struct RayProbe : public madrona::Archetype<RayOrigin, RayDir, RayMaxT, HitEntity, HitT, HitNormal,
                                             RayState> {};
struct Body : public madrona::Archetype<madrona::phys::RigidBody> {};

struct Config {
    madrona::phys::ObjectManager *objMgr;
    uint32_t episodeLen;
    uint32_t uniformBodies;    // 0: from the seed and episode, 8 to variedBodies
    uint32_t variedBodies;     // 0: kVariedMaxBodies
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
    uint32_t variedBodies;
    uint32_t stepInEpisode;
    uint32_t episode;
    float pen;                 // the pen's interior is [-pen, pen]^2
    int32_t numBodies;
    Entity bodies[kMaxBodies];
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
