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
    registry.registerArchetype<Lamp>(ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumLights);

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

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);
    auto spin = builder.addToGraph<ParallelForNode<Engine, spinSystem, Position, Rotation, Spin>>({});
    RenderingSystem::setupTasks(builder, {spin});
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
}

}

MADRONA_BUILD_MWGPU_ENTRY(gallery::Engine, gallery::Sim, gallery::Config, gallery::WorldInit);
