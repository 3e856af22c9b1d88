// Fixture simulator 5 ("gallery", GPU only): the batch ray caster beyond the
// rigid-body fixtures -- per world ~100 renderable props (more than one warp of
// instances: a real per-world TLAS), four mesh types from 2 to 320 triangles
// (a real BLAS), per-instance material / colour overrides, two cameras and two
// lights (a directional light with shadow rays, a spotlight without).  No
// physics: props spin and bob so the TLAS is rebuilt over moving boxes each step.
// The reference's ray caster exists only inside its GPU backend, so there is no
// reference image; tests/test_render_bvh.py checks every pixel against a
// brute-force float64 closest hit over all triangles of the world.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/components.hpp>
#include <madrona/rand.hpp>
#include <madrona/render/ecs.hpp>

namespace gallery {

using madrona::Entity;
using madrona::base::Position;
using madrona::base::Rotation;
using madrona::base::Scale;
using madrona::base::ObjectID;

constexpr int32_t kNumViews = 2;
constexpr int32_t kNumLights = 2;

enum class ExportID : uint32_t {
    PropPos, PropRot, PropScale, PropObj, PropMat, PropColor,
    ViewPos, ViewRot,
    RGB, Depth,
    NumExports,
};

enum class TaskGraphID : uint32_t { Step, NumTaskGraphs };

struct Spin { float phase; };

struct Prop : public madrona::Archetype<
    Position, Rotation, Scale, ObjectID,
    madrona::render::Renderable, madrona::render::MaterialOverride, madrona::render::ColorOverride, Spin
> {};

struct Viewer : public madrona::Archetype<
    Position, Rotation, madrona::render::RenderCamera
> {};

struct Lamp : public madrona::Archetype<
    Position,
    madrona::render::LightDescDirection, madrona::render::LightDescType, madrona::render::LightDescShadow,
    madrona::render::LightDescCutoffAngle, madrona::render::LightDescIntensity, madrona::render::LightDescActive,
    madrona::render::LightCarrier
> {};

struct Config {
    uint32_t numProps;
    uint32_t numMeshes;     // object IDs 0 .. numMeshes - 2 are props, numMeshes - 1 is the ground
};

#if defined(GALLERY_PER_WORLD)
// build variant "gallery_sized": every world says how many props it has (0: not even the
// ground) and how they are laid out
enum class Layout : uint32_t {
    Scattered,      // as the gallery: uniform over the floor
    Clustered,      // a spiral at geometrically shrinking radii and sizes (deep Morton trees)
};
struct WorldInit { uint32_t seed; uint32_t numProps; Layout layout; };
#else
struct WorldInit { uint32_t seed; };
#endif

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
