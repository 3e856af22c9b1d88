// object_manager.h -- layout of the object description a simulator's Config points at
// (== geo::HalfEdge / geo::Plane / geo::HalfEdgeMesh / phys::CollisionPrimitive /
// RigidBodyMetadata / ObjectManager, device/madrona/geo.hpp and device/madrona/physics.hpp).
// physics_assets.cpp builds it, the physics kernels read it.
#pragma once

#include <madrona/math.hpp>

#include <cstdint>

namespace mb2 {

struct HalfEdge {
    uint32_t next;
    uint32_t rootVertex;
    uint32_t face;
};

struct Plane {
    madrona::math::Vector3 normal;
    float d;
};

struct HalfEdgeMesh {
    HalfEdge *halfEdges;
    uint32_t *faceBaseHalfEdges;
    Plane *facePlanes;
    madrona::math::Vector3 *vertices;
    uint32_t numHalfEdges;
    uint32_t numFaces;
    uint32_t numVertices;
};

// CollisionPrimitive::type (== phys::CollisionPrimitive::Type)
constexpr uint32_t kPrimSphere = 1, kPrimHull = 2, kPrimPlane = 4;

struct CollisionPrimitive {
    uint32_t type;     // kPrimSphere, kPrimHull or kPrimPlane
    union {
        float sphereRadius;
        HalfEdgeMesh hull;
    };
};

struct RigidBodyMetadata {
    float invMass;
    madrona::math::Vector3 invInertia;
    madrona::math::Vector3 toCenterOfMass;
    madrona::math::Quat toInertiaFrame;
    float muS;
    float muD;
};

struct ObjectManager {
    CollisionPrimitive *prims;
    madrona::math::AABB *primAABBs;
    madrona::math::AABB *bodyAABBs;
    uint32_t *primOffsets;
    uint32_t *primCounts;
    RigidBodyMetadata *metadata;
};

static_assert(sizeof(CollisionPrimitive) == 56, "CollisionPrimitive layout");
static_assert(sizeof(RigidBodyMetadata) == 52, "RigidBodyMetadata layout");
static_assert(sizeof(ObjectManager) == 48, "ObjectManager layout");

}
