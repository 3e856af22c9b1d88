// Fixture simulator "hullpile": convex hulls at the narrowphase's staging caps, dropped
// into a walled pen -- an octagonal prism (16 vertices, two 8-vertex faces) onto an
// octagonal pedestal, octagonal prisms standing and lying on the floor, an octagonal
// bipyramid (16 faces), tetrahedra, pentagonal pyramids, wedges, boxes, spheres and two
// compound objects in a loose column.  Physics only, no inputs; every world is seeded
// by its index.  Compiled unchanged for the reference CPU backend
// (oracle/harness_hullpile.cpp) and, through NVRTC, for this engine.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/components.hpp>
#include <madrona/physics.hpp>
#include <madrona/rand.hpp>

namespace hullpile {

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

// plane, 4 walls, slab, pedestal, prism on the pedestal, standing and lying prisms,
// a ball sunk into the slab
constexpr int32_t kNumFixed = 11;
#if defined(HULLPILE_MANY)
// build variant: 60 bodies per world, more than the position solve stages in shared
// memory (48), fewer than the candidate search handles (128)
constexpr int32_t kNumColumn = 49;
constexpr float kPen = 6.f;            // pen interior: [-kPen, kPen]^2
#else
constexpr int32_t kNumColumn = 9;
constexpr float kPen = 5.f;
#endif
constexpr int32_t kMaxBodies = kNumFixed + kNumColumn;

enum class ExportID : uint32_t {
    BodyPos,
    BodyRot,
    BodyVel,
    BodyEntity,
    BodyScale,
    BodyObject,
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
    Dumbbell,          // two boxes side by side (two hull primitives)
    CappedBox,         // a box with a sphere primitive on its top face
    Plane,
    Wall,              // static box
    Pedestal,          // static octagonal prism
    NumObjects,
};

// Config::layout
enum class Layout : uint32_t {
    Pile,              // the fixture
    FaceOnFace,        // only an OctPrism upright, base down on an inverted Pedestal
    FaceOnPlane,       // only an OctPrism upright, base down on the plane
};

struct Body : public madrona::Archetype<madrona::phys::RigidBody> {};

struct Config {
    madrona::phys::ObjectManager *objMgr;
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
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
