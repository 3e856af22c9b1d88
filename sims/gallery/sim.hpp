// Fixture simulator 5 ("gallery", GPU only): the batch ray caster beyond the
// rigid-body fixtures -- per world ~100 renderable props (more than one warp of
// instances: a real per-world TLAS), four mesh types from 2 to 320 triangles
// (a real BLAS), per-instance material / colour overrides, two cameras and two
// lights (a directional light with shadow rays, a spotlight without).  No
// physics: props spin and bob so the TLAS is rebuilt over moving boxes each step.
// Built with -DGALLERY_LIGHTS=1 (the "gallery_lit" fixture) each world has its own lamp
// count instead: lamps of every light type among the props, moved and retyped every step
// and respawned every lampPeriod steps, on two carrier archetypes (tests/test_render_lights.py).
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
#if defined(GALLERY_LIGHTS)
constexpr int32_t kNumLights = 12;      // most lamps a world may have (WorldInit numLamps / lampsAfter)
#else
constexpr int32_t kNumLights = 2;
#endif

// PropEntity and Segmentation are exported when built with -DGALLERY_ENTITY_EXPORTS=1, Normals
// when also built with -DGALLERY_NORMAL_EXPORTS=1 (as the fixtures are); without them the
// gallery exports the first ten (or twelve) slots only
enum class ExportID : uint32_t {
    PropPos, PropRot, PropScale, PropObj, PropMat, PropColor,
    ViewPos, ViewRot,
    RGB, Depth,
    PropEntity, Segmentation,
    Normals,
#if defined(GALLERY_LIGHTS)
    // per carrier row, Lamp then Beacon: the light description the ray caster takes from
    // it, the light entity it carries (Entity::none() for none) and its world
    LampPos, LampDir, LampType, LampShadow, LampCutoff, LampLight, LampWorld,
    BeaconPos, BeaconDir, BeaconType, BeaconShadow, BeaconCutoff, BeaconLight, BeaconWorld,
#endif
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

#if defined(GALLERY_LIGHTS)
// what a lamp does each step: circle its anchor, turn its direction about z, flip its shadow
// flag every 3rd and its type every 4th step (offset by its creation index)
struct LampMotion {
    madrona::math::Vector3 anchor;
    float phase, heading, tilt;
    uint32_t index;
};
struct BeaconTag { uint32_t index; };

// a second light carrier archetype: the LightDesc* components in another order, one more
struct Beacon : public madrona::Archetype<
    madrona::render::LightDescActive, madrona::render::LightDescCutoffAngle, BeaconTag,
    madrona::render::LightCarrier, madrona::render::LightDescShadow, LampMotion,
    madrona::render::LightDescIntensity, Position, madrona::render::LightDescType,
    madrona::render::LightDescDirection
> {};

struct LampClock { uint32_t t; };
#endif

struct Lamp : public madrona::Archetype<
    Position,
    madrona::render::LightDescDirection, madrona::render::LightDescType, madrona::render::LightDescShadow,
    madrona::render::LightDescCutoffAngle, madrona::render::LightDescIntensity, madrona::render::LightDescActive,
    madrona::render::LightCarrier
#if defined(GALLERY_LIGHTS)
    , LampMotion
#endif
> {};

struct Config {
    uint32_t numProps;
    uint32_t numMeshes;     // object IDs 0 .. numMeshes - 2 are props, numMeshes - 1 is the ground
#if defined(GALLERY_LIGHTS)
    uint32_t lampPeriod;    // lamps respawn every lampPeriod steps (0: never)
#endif
};

#if defined(GALLERY_PER_WORLD)
// build variant "gallery_sized": every world says how many props it has (0: not even the
// ground) and how they are laid out
enum class Layout : uint32_t {
    Scattered,      // as the gallery: uniform over the floor
    Clustered,      // a spiral at geometrically shrinking radii and sizes (deep Morton trees)
};
struct WorldInit { uint32_t seed; uint32_t numProps; Layout layout; };
#elif defined(GALLERY_LIGHTS)
// build variant "gallery_lit": every world starts with numLamps lamps; each respawn destroys
// every other lamp and creates new ones up to lampsAfter, numLamps, lampsAfter, ... lamps
struct WorldInit { uint32_t seed; uint32_t numLamps; uint32_t lampsAfter; };
#else
struct WorldInit { uint32_t seed; };
#endif

class Engine;

struct Sim : public madrona::WorldBase {
    static void registerTypes(madrona::ECSRegistry &registry, const Config &cfg);
    static void setupTasks(madrona::TaskGraphManager &mgr, const Config &cfg);
    Sim(Engine &ctx, const Config &cfg, const WorldInit &init);
    madrona::RNG rng;
#if defined(GALLERY_LIGHTS)
    uint32_t lampPeriod, numLampsInit, lampsAfter;
    uint32_t respawns, lampsMade, numLamps;
    Entity lamps[kNumLights];
#endif
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
