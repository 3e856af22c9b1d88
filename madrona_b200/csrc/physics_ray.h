// physics_ray.h -- a ray cast against one world's broadphase tree (reference:
// src/physics/broadphase.cpp:658-724, 726-888), shared by two compilers:
//   * NVRTC: broadphase::BVH::traceRay, which simulator code calls (device/madrona/physics.hpp)
//   * nvcc:  the batched ray queries of mb2_trace_physics_rays (physics_rays.cu)
// Both compile it without FMA contraction (--fmad=false, precise division, no flush to zero), so
// a query from the engine returns the bits an in-simulator traceRay returns for the same ray.
#pragma once

#include "physics_state.h"
#include "object_manager.h"

#include <madrona/math.hpp>

namespace mb2::physray {

using madrona::math::Vector3;
using madrona::math::Quat;
using madrona::math::Diag3x3;
using madrona::math::AABB;

__device__ inline bool rayIntoPlane(Vector3 ray_o, Vector3 ray_d, float t_min, float t_max,
                                    float *hit_t, Vector3 *hit_normal)
{
    // object space: the plane is z = 0 with normal +z
    float denom = ray_d.z;
    if (denom == 0) return false;
    float t = -ray_o.z / denom;
    if (t < t_min || t > t_max) return false;
    *hit_t = t;
    *hit_normal = Vector3 { 0, 0, 1 };
    return true;
}

// Ray vs convex polyhedron as an intersection of half-spaces (RTCD 5.3.8);
// face normals point outwards.  A ray that only crosses back faces is a miss.
__device__ inline bool rayIntoHull(const HalfEdgeMesh &mesh, Vector3 ray_o, Vector3 ray_d,
                                   float t_min, float t_max, float *hit_t, Vector3 *hit_normal)
{
    float t_enter = t_min;
    float t_exit = t_max;
    Vector3 enter_normal = Vector3::zero();
    const int32_t num_faces = (int32_t)mesh.numFaces;
    for (int32_t f = 0; f < num_faces; f++) {
        Plane plane = mesh.facePlanes[f];
        float denom = dot(plane.normal, ray_d);
        float neg_dist = plane.d - dot(plane.normal, ray_o);
        if (denom == 0.0f) {
            if (neg_dist < 0.0f) return false;
        } else {
            float t = neg_dist / denom;
            if (denom < 0.0f) {
                if (t >= t_enter) {
                    t_enter = t;
                    enter_normal = plane.normal;
                }
            } else if (t <= t_exit) {
                t_exit = t;
            }
            if (t_enter > t_exit) return false;
        }
    }
    if (enter_normal.x == 0 && enter_normal.y == 0 && enter_normal.z == 0) return false;
    *hit_t = t_enter;
    *hit_normal = enter_normal;
    return true;
}

// The ray against every primitive of leaf leaf_idx, in object space; the world-frame normal of
// the closest hit.  Sphere primitives are skipped (the reference asserts on them).
__device__ inline bool traceRayIntoLeaf(const WorldBVH &bvh, int32_t leaf_idx, Vector3 world_ray_o,
                                        Vector3 world_ray_d, float t_min, float t_max,
                                        float *hit_t, Vector3 *hit_normal)
{
    const ObjectManager *obj_mgr = (const ObjectManager *)bvh.objMgr;
    const int32_t obj = bvh.leafObjIDs[leaf_idx];
    const LeafTransform txfm = bvh.leafTransforms[leaf_idx];
    const Quat rot { txfm.rot.w, txfm.rot.x, txfm.rot.y, txfm.rot.z };
    const Vector3 pos { txfm.pos.x, txfm.pos.y, txfm.pos.z };
    const Quat to_local = rot.inv();

    Vector3 obj_o = to_local.rotateVec(world_ray_o - pos);
    obj_o.x /= txfm.scale.x;
    obj_o.y /= txfm.scale.y;
    obj_o.z /= txfm.scale.z;
    Vector3 obj_d = rot.inv().rotateVec(world_ray_d);
    obj_d.x /= txfm.scale.x;
    obj_d.y /= txfm.scale.y;
    obj_d.z /= txfm.scale.z;
    Diag3x3 inv_d = Diag3x3::fromVec(1.f / obj_d);

    const int32_t prim_offset = (int32_t)obj_mgr->primOffsets[obj];
    const int32_t num_prims = (int32_t)obj_mgr->primCounts[obj];

    Vector3 obj_normal;
    bool hit_leaf = false;
    for (int32_t i = 0; i < num_prims; i++) {
        const int32_t prim_idx = prim_offset + i;
        AABB prim_aabb = obj_mgr->primAABBs[prim_idx];
        if (!prim_aabb.rayIntersects(obj_o, inv_d, 0.f, t_max)) continue;

        const CollisionPrimitive *prim = &obj_mgr->prims[prim_idx];
        bool hit = false;
        if (prim->type == kPrimHull) {
            hit = rayIntoHull(prim->hull, obj_o, obj_d, t_min, t_max, hit_t, &obj_normal);
        } else if (prim->type == kPrimPlane) {
            hit = rayIntoPlane(obj_o, obj_d, t_min, t_max, hit_t, &obj_normal);
        }
        if (hit) {
            hit_leaf = true;
            t_max = *hit_t;
        }
    }
    if (!hit_leaf) return false;
    *hit_normal = rot.rotateVec(obj_normal);
    return true;
}

// The reference's slab test of entry j of an orderedBoxes list against the t_max of that moment:
//   max(mins.x, mins.y, mins.z, 0) <= min(maxes.x, maxes.y, maxes.z, t_max)
// (math.inl:1670-1696, NaN-skipping fminf / fmaxf); *leaf = the entry's leaf index.
__device__ __forceinline__ bool slabEntered(const PVec4 *boxes, int32_t j, Vector3 o, Diag3x3 inv_d,
                                            float t_max, int32_t *leaf)
{
    const PVec4 b0 = boxes[2 * j], b1 = boxes[2 * j + 1];
    const float lx = inv_d.d0 * (b0.x - o.x), ux = inv_d.d0 * (b0.w - o.x);
    const float ly = inv_d.d1 * (b0.y - o.y), uy = inv_d.d1 * (b1.x - o.y);
    const float lz = inv_d.d2 * (b0.z - o.z), uz = inv_d.d2 * (b1.y - o.z);
    const float entry = fmaxf(fminf(lx, ux), fmaxf(fminf(ly, uy), fmaxf(fminf(lz, uz), 0.f)));
    const float exit = fminf(fmaxf(lx, ux), fminf(fmaxf(ly, uy), fminf(fmaxf(lz, uz), t_max)));
    *leaf = __float_as_int(b1.z);
    return entry <= exit;
}

// The closest hit of ray (o, d) within [0, t_max] among the world's leaves: the leaf index, or
// -1 for a miss (*out_t and *out_normal are then not written).  `boxes` holds the world's
// bvh.numTraversal orderedBoxes entries -- bvh.orderedBoxes itself or a copy of it, say in shared
// memory.  Every lane of `peers` calls this together; lanes may trace different worlds.
//
// The reference walks the 4-wide tree with a stack (src/physics/broadphase.cpp:658-724),
// testing child i of a popped node against the t_max current at that moment.  A leaf is entered
// iff its own slot box passes that test when its turn comes: every ancestor box contains it (the
// slab expressions are monotonic in the box bounds and t_max only shrinks), and leaves are met in
// the tree's fixed report order.  So the walk is a linear scan over WorldBVH::orderedBoxes --
// same leaves, same order, same floats, no stack and no node pointer chasing.
//
// Mechanism (results identical by construction): boxes are handled in chunks of 64.
//   1. uniform pass: every lane slab-tests the chunk's boxes against its CURRENT t_max and
//      keeps the passing ones as a 64-bit mask -- all lanes run the same loop, no divergence.
//      t_max only shrinks afterwards and a smaller t_max can only turn a pass into a fail
//      (exit = min(..., t_max)), so the mask is a superset of the leaves the walk enters;
//   2. ordered pass over the mask bits: the slab test is REPEATED with the t_max of that
//      moment -- the reference's exact decision, same expression, same floats -- and the
//      leaves that pass are entered in order.  Each round every lane first moves on to its
//      next entered leaf, then the lanes that called together run the (expensive) leaf
//      test together; the warp votes keep the compiler from folding the two phases back
//      into one divergent loop.
// (The one-phase scan over all boxes spent most of its instructions in the divergent
// "walk to my next entered leaf" loop with most lanes idle.  Seeding t_max with the hit
// of the nearest-entry leaf before the walk is an extra pass over the boxes.)
__device__ inline int32_t traceWorld(const WorldBVH &bvh, const PVec4 *boxes, int32_t num_boxes,
                                     unsigned peers, Vector3 o, Vector3 d, float t_max,
                                     float *out_t, Vector3 *out_normal)
{
    const Diag3x3 inv_d = Diag3x3::fromVec(d).inv();
    int32_t closest = -1;
    Vector3 closest_normal { 0, 0, 0 };

    // (every peer runs the same number of chunk iterations: lanes of one warp may belong to
    // worlds with different leaf counts)
    for (int32_t base = 0; __any_sync(peers, base < num_boxes); base += 64) {
        const int32_t left = num_boxes - base;
        const int32_t chunk = left < 0 ? 0 : (left < 64 ? left : 64);
        unsigned long long cand = 0;
        for (int32_t j = 0; j < chunk; j++) {
            int32_t leaf;
            if (slabEntered(boxes, base + j, o, inv_d, t_max, &leaf)) cand |= 1ull << j;
        }
        while (__any_sync(peers, cand != 0)) {
            int32_t leaf_idx = -1;
            while (cand != 0) {
                const int32_t j = __ffsll((long long)cand) - 1;
                cand &= cand - 1;
                int32_t leaf;
                if (slabEntered(boxes, base + j, o, inv_d, t_max, &leaf)) {
                    leaf_idx = leaf;
                    break;
                }
            }
            __syncwarp(peers);

            if (leaf_idx >= 0) {
                float hit_t;
                Vector3 leaf_normal;
                if (traceRayIntoLeaf(bvh, leaf_idx, o, d, 0.f, t_max, &hit_t, &leaf_normal)) {
                    t_max = hit_t;
                    closest = leaf_idx;
                    closest_normal = leaf_normal;
                }
            }
        }
    }
    if (closest >= 0) {
        *out_t = t_max;
        *out_normal = closest_normal;
    }
    return closest;
}

}
