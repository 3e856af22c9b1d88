#include "sim.hpp"
#include <madrona/mw_gpu_entry.hpp>

using namespace madrona;
using namespace madrona::math;
using namespace madrona::render;

namespace gallery {

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    base::registerTypes(registry);
    RenderingSystem::registerTypes(registry, nullptr);
    registry.registerComponent<Spin>();
    registry.registerArchetype<Prop>();
    registry.registerArchetype<Viewer>(ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumViews);
#if defined(GALLERY_LIGHTS)
    registry.registerComponent<LampMotion>();
    registry.registerComponent<BeaconTag>();
    registry.registerSingleton<LampClock>();
    // a respawn's new rows coexist with the destroyed ones until the compaction
    registry.registerArchetype<Lamp>(ComponentMetadataSelector<> {}, ArchetypeFlags::None, 2 * kNumLights);
    registry.registerArchetype<Beacon>(ComponentMetadataSelector<> {}, ArchetypeFlags::None, 2 * kNumLights + 1);
#else
    registry.registerArchetype<Lamp>(ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumLights);
#endif

    registry.exportColumn<Prop, Position>((uint32_t)ExportID::PropPos);
    registry.exportColumn<Prop, Rotation>((uint32_t)ExportID::PropRot);
    registry.exportColumn<Prop, Scale>((uint32_t)ExportID::PropScale);
    registry.exportColumn<Prop, ObjectID>((uint32_t)ExportID::PropObj);
    registry.exportColumn<Prop, MaterialOverride>((uint32_t)ExportID::PropMat);
    registry.exportColumn<Prop, ColorOverride>((uint32_t)ExportID::PropColor);
    registry.exportColumn<Viewer, Position>((uint32_t)ExportID::ViewPos);
    registry.exportColumn<Viewer, Rotation>((uint32_t)ExportID::ViewRot);
    registry.exportColumn<RaycastOutputArchetype, RGBOutputBuffer>((uint32_t)ExportID::RGB);
    registry.exportColumn<RaycastOutputArchetype, DepthOutputBuffer>((uint32_t)ExportID::Depth);
#if defined(GALLERY_ENTITY_EXPORTS)
    registry.exportColumn<Prop, Entity>((uint32_t)ExportID::PropEntity);
    registry.exportColumn<RaycastOutputArchetype, SegmentationOutputBuffer>((uint32_t)ExportID::Segmentation);
#if defined(GALLERY_NORMAL_EXPORTS)
    registry.exportColumn<RaycastOutputArchetype, NormalOutputBuffer>((uint32_t)ExportID::Normals);
#endif
#endif
#if defined(GALLERY_LIGHTS)
    registry.exportColumn<Lamp, Position>((uint32_t)ExportID::LampPos);
    registry.exportColumn<Lamp, LightDescDirection>((uint32_t)ExportID::LampDir);
    registry.exportColumn<Lamp, LightDescType>((uint32_t)ExportID::LampType);
    registry.exportColumn<Lamp, LightDescShadow>((uint32_t)ExportID::LampShadow);
    registry.exportColumn<Lamp, LightDescCutoffAngle>((uint32_t)ExportID::LampCutoff);
    registry.exportColumn<Lamp, LightCarrier>((uint32_t)ExportID::LampLight);
    registry.exportColumn<Lamp, WorldID>((uint32_t)ExportID::LampWorld);
    registry.exportColumn<Beacon, Position>((uint32_t)ExportID::BeaconPos);
    registry.exportColumn<Beacon, LightDescDirection>((uint32_t)ExportID::BeaconDir);
    registry.exportColumn<Beacon, LightDescType>((uint32_t)ExportID::BeaconType);
    registry.exportColumn<Beacon, LightDescShadow>((uint32_t)ExportID::BeaconShadow);
    registry.exportColumn<Beacon, LightDescCutoffAngle>((uint32_t)ExportID::BeaconCutoff);
    registry.exportColumn<Beacon, LightCarrier>((uint32_t)ExportID::BeaconLight);
    registry.exportColumn<Beacon, WorldID>((uint32_t)ExportID::BeaconWorld);
#endif
}

// props turn about z by a fixed small step (cos, sin of 0.02 rad as literals) and bob
inline void spinSystem(Engine &, Position &pos, Rotation &rot, Spin &spin)
{
    const Quat dq { 0.99995f, 0.f, 0.f, 0.0099998f };
    Quat q = rot;
    rot = (dq * q).normalize();
    spin.phase += 0.05f;
    if (spin.phase > 1.f) spin.phase -= 2.f;
    pos.z += 0.01f * spin.phase;
}

#if defined(GALLERY_LIGHTS)
// a lamp of a random kind (directional, spotlight with a 0.3 - 1.3 rad cone, or point light:
// a spotlight with cutoff -1), shadow flag, intensity and active flag, anchored among the props
// (whose centres lie 0.6 - 3.1 above the floor) or above them, pointing down at a tilt
template <typename ArchetypeT>
static Entity makeLampOf(Engine &ctx, Sim &sim)
{
    Entity e = ctx.makeEntity<ArchetypeT>();
    if (e.id < 0) return e;
    RNG &rng = sim.rng;
    const int32_t kind = rng.sampleI32(0, 3);
    LampMotion m;
    m.anchor = Vector3 { (rng.sampleUniform() - 0.5f) * 20.f, (rng.sampleUniform() - 0.5f) * 20.f,
                         0.8f + 5.f * rng.sampleUniform() };
    m.phase = 6.2831853f * rng.sampleUniform();
    m.heading = 6.2831853f * rng.sampleUniform();
    m.tilt = 0.15f + 0.75f * rng.sampleUniform();
    m.index = sim.lampsMade++;
    ctx.get<LampMotion>(e) = m;
    ctx.get<Position>(e) = m.anchor;
    ctx.get<LightDescDirection>(e) =
        LightDescDirection(Vector3 { m.tilt * cosf(m.heading), m.tilt * sinf(m.heading), -1.f }.normalize());
    ctx.get<LightDescType>(e).type = kind == 0 ? LightDesc::Directional : LightDesc::Spotlight;
    ctx.get<LightDescShadow>(e).castShadow = rng.sampleBool();
    const float cone = 0.3f + rng.sampleUniform();
    ctx.get<LightDescCutoffAngle>(e).cutoff = kind == 2 ? -1.f : cone;
    ctx.get<LightDescIntensity>(e).intensity = 0.25f + 1.75f * rng.sampleUniform();
    ctx.get<LightDescActive>(e).active = rng.sampleUniform() < 0.75f;
    RenderingSystem::makeEntityLightCarrier(ctx, e);
    return e;
}

// every third lamp a world makes is a Beacon
static Entity makeLamp(Engine &ctx, Sim &sim)
{
    if (sim.lampsMade % 3 == 1) {
        const uint32_t index = sim.lampsMade;
        Entity e = makeLampOf<Beacon>(ctx, sim);
        if (e.id >= 0) ctx.get<BeaconTag>(e).index = index;
        return e;
    }
    return makeLampOf<Lamp>(ctx, sim);
}

static void destroyLamp(Engine &ctx, Entity lamp)
{
    const Entity light = ctx.get<LightCarrier>(lamp).light;
    if (light.id >= 0) ctx.destroyEntity(light);
    ctx.destroyEntity(lamp);
}

inline void lampClockSystem(Engine &, LampClock &c)
{
    c.t += 1;
}

// lamps of both carrier archetypes: circle the anchor, turn, flip shadow flag and type now and then
inline void lampSystem(Engine &ctx, Position &pos, LightDescDirection &dir, LightDescType &type,
                       LightDescShadow &shadow, LampMotion &m)
{
    const uint32_t t = ctx.singleton<LampClock>().t + m.index;
    m.phase += 0.35f;
    m.heading += 0.25f;
    pos = m.anchor + Vector3 { 1.2f * cosf(m.phase), 1.2f * sinf(m.phase), 0.4f * sinf(0.7f * m.phase) };
    dir = LightDescDirection(Vector3 { m.tilt * cosf(m.heading), m.tilt * sinf(m.heading), -1.f }.normalize());
    if (t % 3 == 0) shadow.castShadow = !shadow.castShadow;
    if (t % 4 == 0) {
        type.type = type.type == LightDesc::Directional ? LightDesc::Spotlight : LightDesc::Directional;
    }
}

// one thread per world: every lampPeriod steps, destroy every other lamp (with its light
// entity) and any past the new count, then make lamps up to it
inline void lampRespawnSystem(Engine &ctx, LampClock &c)
{
    Sim &sim = ctx.data();
    if (sim.lampPeriod == 0 || c.t % sim.lampPeriod != 0) return;
    sim.respawns++;
    const uint32_t target = (sim.respawns & 1) ? sim.lampsAfter : sim.numLampsInit;
    uint32_t kept = 0;
    for (uint32_t i = 0; i < sim.numLamps; i++) {
        if (i % 2 == 0 || kept >= target) {
            destroyLamp(ctx, sim.lamps[i]);
        } else {
            sim.lamps[kept++] = sim.lamps[i];
        }
    }
    while (kept < target) sim.lamps[kept++] = makeLamp(ctx, sim);
    sim.numLamps = kept;
}
#endif

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);
    auto spin = builder.addToGraph<ParallelForNode<Engine, spinSystem, Position, Rotation, Spin>>({});
#if defined(GALLERY_LIGHTS)
    auto clock = builder.addToGraph<ParallelForNode<Engine, lampClockSystem, LampClock>>({spin});
    auto move = builder.addToGraph<ParallelForNode<Engine, lampSystem, Position, LightDescDirection, LightDescType,
                                                   LightDescShadow, LampMotion>>({clock});
    auto respawn = builder.addToGraph<ParallelForNode<Engine, lampRespawnSystem, LampClock>>({move});
    auto lamps = builder.addToGraph<CompactArchetypeNode<Lamp>>({respawn});
    auto beacons = builder.addToGraph<CompactArchetypeNode<Beacon>>({lamps});
    RenderingSystem::setupTasks(builder, {beacons});
#else
    RenderingSystem::setupTasks(builder, {spin});
#endif
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx), rng(init.seed)
{
    RenderingSystem::init(ctx, nullptr);
    const uint32_t ground_obj = cfg.numMeshes - 1;
#if defined(GALLERY_PER_WORLD)
    const uint32_t num_props = init.numProps;
    const bool clustered = init.layout == Layout::Clustered;
#else
    const uint32_t num_props = cfg.numProps;
    const bool clustered = false;
#endif

    // the ground: one big quad
    if (num_props > 0) {
        Entity e = ctx.makeEntity<Prop>();
        ctx.get<Position>(e) = Vector3 { 0, 0, 0 };
        ctx.get<Rotation>(e) = Quat { 1, 0, 0, 0 };
        ctx.get<Scale>(e) = Diag3x3 { 1, 1, 1 };
        ctx.get<ObjectID>(e) = ObjectID { (int32_t)ground_obj };
        ctx.get<MaterialOverride>(e).matID = 0;
        ctx.get<ColorOverride>(e).color = 0xFFFFFFu;
        ctx.get<Spin>(e).phase = 0.f;
        RenderingSystem::makeEntityRenderable(ctx, e);
    }
    for (uint32_t i = 1; i < num_props; i++) {
        Entity e = ctx.makeEntity<Prop>();
        float x = (rng.sampleUniform() - 0.5f) * 24.f;
        float y = (rng.sampleUniform() - 0.5f) * 24.f;
        float z = 0.6f + rng.sampleUniform() * 2.5f;
        float s = 0.5f + rng.sampleUniform();
        if (clustered) {
            // prop i sits at radius 6 * 0.93^i around (0, 0, 2), at 1/8 of that size
            const float r = 6.f * powf(0.93f, (float)i);
            const float a = 2.39996f * (float)i;
            x = r * cosf(a);
            y = r * sinf(a);
            z = 2.f + 0.3f * r;
            s = 0.125f * r;
        }
        ctx.get<Position>(e) = Vector3 { x, y, z };
        Quat q { rng.sampleUniform() - 0.5f, rng.sampleUniform() - 0.5f, rng.sampleUniform() - 0.5f,
                 rng.sampleUniform() + 0.1f };
        ctx.get<Rotation>(e) = q.normalize();
        ctx.get<Scale>(e) = Diag3x3 { s, s * (0.6f + 0.8f * rng.sampleUniform()), s };
        ctx.get<ObjectID>(e) = ObjectID { rng.sampleI32(0, (int32_t)ground_obj) };
        // a third each: mesh default material, material override, colour override
        int32_t mode = rng.sampleI32(0, 3);
        ctx.get<MaterialOverride>(e).matID = mode == 0 ? -1 : (mode == 1 ? rng.sampleI32(0, 4) : -2);
        ctx.get<ColorOverride>(e).color = (uint32_t)rng.sampleI32(0, 0x1000000);
        ctx.get<Spin>(e).phase = rng.sampleUniform() - 0.5f;
        RenderingSystem::makeEntityRenderable(ctx, e);
        // every 17th prop is hidden again
        if (i % 17 == 0) RenderingSystem::disableEntityRenderable(ctx, e);
    }

    for (int32_t v = 0; v < kNumViews; v++) {
        Entity e = ctx.makeEntity<Viewer>();
        float a = rng.sampleUniform();
        ctx.get<Position>(e) = v == 0 ? Vector3 { -14.f + a, -14.f, 4.f } : Vector3 { 13.f, 2.f * a, 2.f };
        // looking towards the middle: yaw 45 degrees left / 90 degrees left, pitched a little down
        Quat yaw = v == 0 ? Quat { 0.92387953f, 0, 0, -0.38268343f } : Quat { 0.70710678f, 0, 0, 0.70710678f };
        Quat pitch { 0.9961947f, -0.0871557f, 0, 0 };
        ctx.get<Rotation>(e) = (yaw * pitch).normalize();
        RenderingSystem::attachEntityToView(ctx, e, 70.f, 0.001f, Vector3 { 0.f, 0.f, 0.25f });
    }

#if defined(GALLERY_LIGHTS)
    lampPeriod = cfg.lampPeriod;
    numLampsInit = init.numLamps < (uint32_t)kNumLights ? init.numLamps : (uint32_t)kNumLights;
    lampsAfter = init.lampsAfter < (uint32_t)kNumLights ? init.lampsAfter : (uint32_t)kNumLights;
    respawns = 0;
    lampsMade = 0;
    ctx.singleton<LampClock>().t = 0;
    for (numLamps = 0; numLamps < numLampsInit; numLamps++) lamps[numLamps] = makeLamp(ctx, *this);
    // a carrier that carries no light: the light refresh must pass it by
    {
        Entity e = ctx.makeEntity<Beacon>();
        ctx.get<Position>(e) = Vector3 { 0.f, 0.f, 5.f };
        ctx.get<LightDescDirection>(e) = LightDescDirection(Vector3 { 0.f, 0.f, -1.f });
        ctx.get<LightDescType>(e).type = LightDesc::Directional;
        ctx.get<LightDescShadow>(e).castShadow = false;
        ctx.get<LightDescCutoffAngle>(e).cutoff = 0.5f;
        ctx.get<LightDescIntensity>(e).intensity = 1.f;
        ctx.get<LightDescActive>(e).active = true;
        ctx.get<LampMotion>(e) = LampMotion { Vector3 { 0.f, 0.f, 5.f }, 0.f, 0.f, 0.5f, 0u };
        ctx.get<BeaconTag>(e).index = 0xFFFFFFFFu;
        ctx.get<LightCarrier>(e).light = Entity::none();
    }
#else
    for (int32_t l = 0; l < kNumLights; l++) {
        Entity e = ctx.makeEntity<Lamp>();
        ctx.get<Position>(e) = Vector3 { 0.f, 0.f, 9.f };
        Vector3 dir = l == 0 ? Vector3 { 0.3f, 0.2f, -0.9327379f } : Vector3 { 0.f, 0.f, -1.f };
        ctx.get<LightDescDirection>(e) = LightDescDirection(dir);
        ctx.get<LightDescType>(e).type = l == 0 ? LightDesc::Directional : LightDesc::Spotlight;
        ctx.get<LightDescShadow>(e).castShadow = l == 0;
        ctx.get<LightDescCutoffAngle>(e).cutoff = 0.9f;
        ctx.get<LightDescIntensity>(e).intensity = 1.f;
        ctx.get<LightDescActive>(e).active = true;
        RenderingSystem::makeEntityLightCarrier(ctx, e);
    }
#endif
}

}

MADRONA_BUILD_MWGPU_ENTRY(gallery::Engine, gallery::Sim, gallery::Config, gallery::WorldInit);
