#include "sim.hpp"

#ifdef MADRONA_GPU_MODE
#include <madrona/mw_gpu_entry.hpp>
#endif

using namespace madrona;
using namespace madrona::math;
using namespace madrona::phys;

namespace hullpile {

constexpr float kDeltaT = 0.04f;
constexpr CountT kNumSubsteps = 4;
constexpr float kWallThick = 0.5f;
constexpr float kWallHeight = 6.f;

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    base::registerTypes(registry);
    PhysicsSystem::registerTypes(registry);

    registry.registerArchetype<Body>();

    registry.exportColumn<Body, Position>((uint32_t)ExportID::BodyPos);
    registry.exportColumn<Body, Rotation>((uint32_t)ExportID::BodyRot);
    registry.exportColumn<Body, Velocity>((uint32_t)ExportID::BodyVel);
    registry.exportColumn<Body, Entity>((uint32_t)ExportID::BodyEntity);
    // what a body is, for tests/hull_contact_model.py
    registry.exportColumn<Body, Scale>((uint32_t)ExportID::BodyScale);
    registry.exportColumn<Body, ObjectID>((uint32_t)ExportID::BodyObject);
}

static inline Entity makeBody(Engine &ctx, Vector3 pos, Quat rot, Diag3x3 scale,
                              SimObject obj, ResponseType resp)
{
    Entity e = ctx.makeEntity<Body>();
    ObjectID obj_id { (int32_t)obj };
    ctx.get<Position>(e) = pos;
    ctx.get<Rotation>(e) = rot;
    ctx.get<Scale>(e) = scale;
    ctx.get<ObjectID>(e) = obj_id;
    ctx.get<ResponseType>(e) = resp;
    ctx.get<Velocity>(e) = Velocity { Vector3::zero(), Vector3::zero() };
    ctx.get<ExternalForce>(e) = Vector3::zero();
    ctx.get<ExternalTorque>(e) = Vector3::zero();
    ctx.get<broadphase::LeafID>(e) = PhysicsSystem::registerEntity(ctx, e, obj_id);
    return e;
}

// yaw only: normalised (1, 0, 0, s), a turn of 2 atan(s) about +z
static inline Quat yawQuat(float s)
{
    return Quat { 1.f, 0.f, 0.f, s }.normalize();
}

// any orientation: four uniform samples, normalised
static inline Quat randomQuat(RNG &rng)
{
    float w = rng.sampleUniform() - 0.5f;
    float x = rng.sampleUniform() - 0.5f;
    float y = rng.sampleUniform() - 0.5f;
    float z = rng.sampleUniform() - 0.5f;
    return Quat { w, x, y, z }.normalize();
}

// the objects of the column, in turn
static constexpr SimObject kColumn[] = {
    SimObject::Bipyramid, SimObject::Box, SimObject::Dumbbell, SimObject::Tetra,
    SimObject::CappedBox, SimObject::PentaPyramid, SimObject::Wedge, SimObject::Ball,
    SimObject::OctPrism, SimObject::Bipyramid, SimObject::Dumbbell,
};
constexpr int32_t kColumnKinds = sizeof(kColumn) / sizeof(kColumn[0]);

static void makePile(Engine &ctx, RNG &rng)
{
    const Quat upright { 1, 0, 0, 0 };

    // four walls around the pen and a slab lying on the floor, static boxes
    const float reach = kPen + kWallThick;
    const float mid = kPen + 0.5f * kWallThick;
    makeBody(ctx, Vector3 { 0, -mid, 0.5f * kWallHeight }, upright,
             Diag3x3 { 2.f * reach, kWallThick, kWallHeight }, SimObject::Wall, ResponseType::Static);
    makeBody(ctx, Vector3 { 0, mid, 0.5f * kWallHeight }, upright,
             Diag3x3 { 2.f * reach, kWallThick, kWallHeight }, SimObject::Wall, ResponseType::Static);
    makeBody(ctx, Vector3 { -mid, 0, 0.5f * kWallHeight }, upright,
             Diag3x3 { kWallThick, 2.f * kPen, kWallHeight }, SimObject::Wall, ResponseType::Static);
    makeBody(ctx, Vector3 { mid, 0, 0.5f * kWallHeight }, upright,
             Diag3x3 { kWallThick, 2.f * kPen, kWallHeight }, SimObject::Wall, ResponseType::Static);
    makeBody(ctx, Vector3 { -2.5f, 2.5f, 0.25f }, yawQuat(0.3f), Diag3x3 { 3.f, 2.f, 0.5f },
             SimObject::Wall, ResponseType::Static);

    // an octagonal prism dropped flat onto an octagonal pedestal of the same width at a
    // yaw between 11 and 33 degrees: an 8-gon clipped against an 8-gon (16 points)
    // (one random sample per statement: argument evaluation order is unspecified)
    makeBody(ctx, Vector3 { 2.5f, 2.5f, 0.5f }, upright, Diag3x3 { 1.6f, 1.6f, 1.f },
             SimObject::Pedestal, ResponseType::Static);
    const float drop = 1.6f + 0.3f * rng.sampleUniform();
    const float turn = 0.1f + 0.2f * rng.sampleUniform();
    makeBody(ctx, Vector3 { 2.5f, 2.5f, drop }, yawQuat(turn), Diag3x3 { 1.6f, 1.6f, 0.6f },
             SimObject::OctPrism, ResponseType::Dynamic);

    // octagonal prisms on the floor: standing (an 8-vertex face on the plane) and lying
    const float stand_turn = 0.1f + 0.3f * rng.sampleUniform();
    makeBody(ctx, Vector3 { -2.5f, -2.5f, 0.45f }, yawQuat(stand_turn),
             Diag3x3 { 1.2f, 1.2f, 0.8f }, SimObject::OctPrism, ResponseType::Dynamic);
    makeBody(ctx, Vector3 { 1.f, -3.f, 0.8f }, Quat { 1, 1, 0, 0 }.normalize(),
             Diag3x3 { 1.2f, 1.2f, 1.5f }, SimObject::OctPrism, ResponseType::Dynamic);

    // a ball whose centre starts inside the slab, pushed out through sphere - hull contacts
    const float ball_x = -2.5f + 0.4f * rng.sampleUniform();
    makeBody(ctx, Vector3 { ball_x, 2.5f, 0.4f }, upright,
             Diag3x3 { 1.f, 1.f, 1.f }, SimObject::Ball, ResponseType::Dynamic);

    // the column: random orientations, non-uniform scales on hulls (uniform on anything
    // with a sphere), stacks of six at up to nine spots 2.6 m apart; levels 2.4 m apart,
    // the lowest clear of the prism on the pedestal, so that nothing overlaps at step 0
    for (int32_t i = 0; i < kNumColumn; i++) {
        const SimObject obj = kColumn[i % kColumnKinds];
        const int32_t spot = i / 6;
        const int32_t level = i % 6;
        float x = 2.6f * (float)(spot % 3 - 1) + 0.8f * (rng.sampleUniform() - 0.5f);
        float y = 2.6f * (float)(spot / 3 - 1) + 0.8f * (rng.sampleUniform() - 0.5f);
        float z = 3.5f + 2.4f * (float)level;
        Diag3x3 scale { 1.f, 1.f, 1.f };
        if (obj != SimObject::Ball && obj != SimObject::CappedBox) {
            scale.d0 = 0.7f + 0.6f * rng.sampleUniform();
            scale.d1 = 0.7f + 0.6f * rng.sampleUniform();
            scale.d2 = 0.7f + 0.6f * rng.sampleUniform();
        }
        makeBody(ctx, Vector3 { x, y, z }, randomQuat(rng), scale, obj, ResponseType::Dynamic);
    }
}

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &builder = mgr.init(TaskGraphID::Step);
    auto broadphase = PhysicsSystem::setupBroadphaseTasks(builder, {});
    auto physics = PhysicsSystem::setupPhysicsStepTasks(builder, {broadphase},
                                                        kNumSubsteps);
    PhysicsSystem::setupCleanupTasks(builder, {physics});
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx),
      rng(init.seed)
{
    PhysicsSystem::init(ctx, cfg.objMgr, kDeltaT, kNumSubsteps,
                        -9.8f * math::up, kMaxBodies);
    PhysicsSystem::reset(ctx);

    const Quat upright { 1, 0, 0, 0 };
    makeBody(ctx, Vector3 { 0, 0, 0 }, upright, Diag3x3 { 1, 1, 1 }, SimObject::Plane,
             ResponseType::Static);

    // Both other layouts rest an OctPrism's local -z face (z = -0.5) on something at step
    // 0, 1 cm deep, for objects that replace the prism with a hull of a bigger base.
    switch ((Layout)cfg.layout) {
    case Layout::FaceOnFace:
        // on the -z face of a Pedestal turned upside down (that face at z = 1.5), a
        // relative yaw of pi / 11
        makeBody(ctx, Vector3 { 0, 0, 1.f }, Quat { 0, 1, 0, 0 }, Diag3x3 { 1, 1, 1 },
                 SimObject::Pedestal, ResponseType::Static);
        makeBody(ctx, Vector3 { 0, 0, 1.99f }, yawQuat(0.14383695f), Diag3x3 { 1, 1, 1 },
                 SimObject::OctPrism, ResponseType::Dynamic);
        break;
    case Layout::FaceOnPlane:
        makeBody(ctx, Vector3 { 0, 0, 0.49f }, upright, Diag3x3 { 1, 1, 1 },
                 SimObject::OctPrism, ResponseType::Dynamic);
        break;
    default:
        makePile(ctx, rng);
        break;
    }
}

}

#ifdef MADRONA_GPU_MODE
MADRONA_BUILD_MWGPU_ENTRY(hullpile::Engine, hullpile::Sim, hullpile::Config, hullpile::WorldInit);
#endif
