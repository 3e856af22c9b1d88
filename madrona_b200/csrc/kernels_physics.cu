// kernels_physics.cu -- hot system 2: rigid-body physics for every world of the
// batch, as ahead-of-time sm_90a kernels over the ECS SoA columns.
//
// WHAT is computed follows the reference's CPU backend so results can be
// compared number for number (SURVEY.md 9.5-9.7):
//   broadphase  src/physics/broadphase.cpp:47-285 (top-down 4-wide midpoint
//               build, only on reset), :440-485 (leaf boxes grown by motion),
//               :550-647 (grow-only refit), :930-993 (pair emission order)
//   narrowphase src/physics/narrowphase.cpp:151-223, 339-365, 464-567, 617-652,
//               659-768, 771-1138, 1214-1514, 1682-1899 (scalar SAT path --
//               the warp-cooperative variant is dead code there, SURVEY F4)
//   XPBD        src/physics/xpbd.cpp:100-185, 454-550, 607-718, 720-779,
//               916-1052
// HOW it runs is new:
//   * candidates and contacts are flat per-world segments written in the CPU
//     backend's iteration order by warp-per-world kernels (count -> warp scan ->
//     emit; ballot-compaction for contacts).  The reference GPU backend
//     appends them with global atomics in racy order and then needs a full
//     radix sort of the Contact and Joint archetypes every substep; here order
//     is deterministic by construction and those ~8 sorts disappear.
//   * every kernel reads the component columns straight from the table
//     descriptors (coalesced AoS-in-SoA rows), no per-row Context / hash lookup.
//   * IEEE arithmetic (--fmad=false) and the reference's operation order, so
//     floats track the CPU oracle.
#include "physics_host.hpp"
#include "physics_state.h"
#include "object_manager.h"

#include <madrona/math.hpp>
#include <madrona/gjk.hpp>

#include <cfloat>
#include <algorithm>

namespace mb2 {

using madrona::math::Vector3;
using madrona::math::Vector4;
using madrona::math::Quat;
using madrona::math::Diag3x3;
using madrona::math::Mat3x3;
using madrona::math::AABB;
using madrona::math::cross;
using madrona::math::dot;

static_assert(sizeof(BVHNode) == 116, "BVH node layout");
static_assert(sizeof(Contact) == 112, "contact layout");
static_assert(sizeof(Candidate) == 32, "candidate layout");

struct PVelocity {
    Vector3 linear;
    Vector3 angular;
};

struct PPosRot {        // SubstepPrevState / PreSolvePositional
    Vector3 x;
    Quat q;
};

struct PJoint {         // == phys::JointConstraint (92 bytes)
    u32 e1Gen; i32 e1ID;
    u32 e2Gen; i32 e2ID;
    i32 type;           // 0 fixed, 1 hinge
    union {
        struct { Quat attachRot1; Quat attachRot2; float separation; } fixed;
        struct { Vector3 a1Local, a2Local, b1Local, b2Local; } hinge;
    };
    Vector3 r1;
    Vector3 r2;
};
static_assert(sizeof(PJoint) == 92, "JointConstraint layout");

constexpr u32 kRespDynamic = 0, kRespStatic = 2;
constexpr int kPhysWarps = 2;     // worlds (warps) per block of the per-world physics kernels

struct PhysicsHost {
    PhysicsState *dPhys = nullptr;
    PhysicsState hPhys;
    bool active = false;
    bool spheres = false;     // some registered object has a sphere primitive (read before graph capture)
    unsigned narrowBlocks = 0;   // persistent narrowphase grid for that kernel (0: occupancy query failed)
    // hulls past the staging caps (MADRONA_B200_MAX_HULL_SIZE > 16)
    i32 *classInfo = nullptr;        // device scratch of the primitive classification
    unsigned char *primClass = nullptr;
    i32 primClassCapacity = 0;
    bool largeHulls = false;         // some primitive needs the warp-per-pair kernel (read before graph capture)
    unsigned largeBlocks = 0;        // its persistent grid (0: it does not fit / the query failed)
    std::string largeError;          // why a launch graph with physics cannot be built
    // worlds past 128 bodies (MADRONA_B200_MAX_BODIES_PER_WORLD > 128)
    unsigned largeSearchBlocks = 0;  // persistent grid of physFindCandidatesLargeKernel (0: query failed)
};

// ---- small device helpers ------------------------------------------------------------

__device__ __forceinline__ const BodyArchetype *bodyOf(const PhysicsState &P, u32 arch)
{
    if (arch >= (u32)kMaxArchetypes) return nullptr;
    const int idx = P.bodyIndex[arch];
    return idx < 0 ? nullptr : &P.bodies[idx];
}

template <typename T>
__device__ __forceinline__ T &bodyCol(const EngineState &S, const BodyArchetype &b, int pc, i32 row)
{
    return ((T *)S.tables[b.archetype].columns[b.cols[pc]])[row];
}

// Column base pointers of every (rigid-body archetype, physics component), staged in shared
// memory by each per-world / per-candidate kernel before its first access (fillColCache).
// A component access by (archetype id, row) is then one shared-memory lookup and one global
// load; through PhysicsState::bodyIndex -> bodies[].cols -> tables[].columns it was a chain
// of three dependent global loads before the data (ncu, position solve: 37 % of the stall
// samples sat on that chain).  Sorts flip column pointers only between kernels.
struct ColCache {
    void *ptr[kMaxBodyArchetypes][PCCount];
    signed char bodyIndex[kMaxArchetypes];
};
__shared__ ColCache g_cols;

__device__ __forceinline__ void fillColCache(const EngineState &S, const PhysicsState &P)
{
    const int n = (int)P.numBodyArchetypes * (int)PCCount;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int bi = i / (int)PCCount, pc = i - bi * (int)PCCount;
        const BodyArchetype &b = P.bodies[bi];
        const i32 col = b.cols[pc];
        g_cols.ptr[bi][pc] = col >= 0 ? S.tables[b.archetype].columns[col] : nullptr;
    }
    for (int i = threadIdx.x; i < kMaxArchetypes; i += blockDim.x) g_cols.bodyIndex[i] = P.bodyIndex[i];
    __syncthreads();
}

__device__ __forceinline__ bool isBodyArchetype(u32 arch)
{
    return arch < (u32)kMaxArchetypes && g_cols.bodyIndex[arch] >= 0;
}

// Component `pc` of row `row` of body archetype `arch`; fillColCache must have run in the block.
template <typename T>
__device__ __forceinline__ T &cachedCol(u32 arch, int pc, i32 row)
{
    return ((T *)g_cols.ptr[g_cols.bodyIndex[arch]][pc])[row];
}

__device__ __forceinline__ WorldBVH &worldBVH(const EngineState &S, const PhysicsState &P, i32 w)
{
    return ((WorldBVH *)S.tables[P.bvhArchetype].columns[2])[w];
}

__device__ __forceinline__ const PhysicsWorldParams &worldParams(const EngineState &S, const PhysicsState &P, i32 w)
{
    return ((const PhysicsWorldParams *)S.tables[P.paramsArchetype].columns[2])[w];
}

__device__ __forceinline__ const ObjectManager &worldObjects(const EngineState &S, const PhysicsState &P, i32 w)
{
    return **(const ObjectManager *const *)((const char *)S.tables[P.objectDataArchetype].columns[2] +
                                            (size_t)w * 8);
}

__device__ __forceinline__ Vector3 mulDiag(Vector3 d, Vector3 v)
{
    return Vector3 { d.x * v.x, d.y * v.y, d.z * v.z };
}

// Wide accesses for the 16 / 24 / 40-byte row types (columns are 256-byte
// aligned, BVH arrays 128-byte aligned): one request per 8 or 16 bytes instead
// of one per float -- the row kernels are LSU-queue bound otherwise.
__device__ __forceinline__ Quat loadQuat(const Quat *p)
{
    const float4 v = *reinterpret_cast<const float4 *>(p);
    return Quat { v.x, v.y, v.z, v.w };
}

__device__ __forceinline__ void storeQuat(Quat *p, Quat q)
{
    *reinterpret_cast<float4 *>(p) = make_float4(q.w, q.x, q.y, q.z);
}

template <typename T>
__device__ __forceinline__ T loadPairs(const T *p)
{
    static_assert(sizeof(T) % 8 == 0, "");
    union { T t; float2 v[sizeof(T) / 8]; } u;
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 8); i++) u.v[i] = reinterpret_cast<const float2 *>(p)[i];
    return u.t;
}

template <typename T>
__device__ __forceinline__ void storePairs(T *p, const T &value)
{
    static_assert(sizeof(T) % 8 == 0, "");
    union U { T t; float2 v[sizeof(T) / 8]; __device__ U() {} } u;
    u.t = value;
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 8); i++) reinterpret_cast<float2 *>(p)[i] = u.v[i];
}

// Float min / max as ONE native integer atomic (no CAS loop, no return value needed): for
// value >= 0 the signed-int order of the bit patterns is the float order (every negative float
// is a negative int), for value < 0 the unsigned order is the reversed float order.
__device__ __forceinline__ void atomicMinFloat(float *addr, float value)
{
    if (value >= 0.f) atomicMin((int *)addr, __float_as_int(value));
    else atomicMax((unsigned int *)addr, __float_as_uint(value));
}

__device__ __forceinline__ void atomicMaxFloat(float *addr, float value)
{
    if (value >= 0.f) atomicMax((int *)addr, __float_as_int(value));
    else atomicMin((unsigned int *)addr, __float_as_uint(value));
}

// =============================================================================================
// Broadphase
// =============================================================================================

// Leaf box = object box under TRS, stretched along the motion of the next
// step: per axis delta = velExpansion * v, min += delta - a if negative,
// max += delta + a if positive (broadphase.cpp:440-464).
__device__ __forceinline__ AABB growByMotion(AABB box, Vector3 v, float vel_k, float accel_k)
{
    for (int i = 0; i < 3; i++) {
        float delta = vel_k * v[i];
        float lo = delta - accel_k;
        float hi = delta + accel_k;
        if (lo < 0.f) box.pMin[i] += lo;
        if (hi > 0.f) box.pMax[i] += hi;
    }
    return box;
}

__device__ __forceinline__ void rowUpdateLeaf(const EngineState &S, const PhysicsState &P, const BodyArchetype &b, const i32 row, const i32 w)
{
    {
        WorldBVH &bvh = worldBVH(S, P, w);
        const ObjectManager &objs = *(const ObjectManager *)bvh.objMgr;

        const i32 leaf = bodyCol<i32>(S, b, PCLeafID, row);
        const Vector3 pos = bodyCol<Vector3>(S, b, PCPosition, row);
        const Quat rot = loadQuat(&bodyCol<Quat>(S, b, PCRotation, row));
        const Diag3x3 scale = bodyCol<Diag3x3>(S, b, PCScale, row);
        const i32 obj = bodyCol<i32>(S, b, PCObjectID, row);
        const Vector3 lin_vel = bodyCol<PVelocity>(S, b, PCVelocity, row).linear;

        AABB world_box = objs.bodyAABBs[obj].applyTRS(pos, rot, scale);
        AABB grown = growByMotion(world_box, lin_vel, bvh.velExpansion, bvh.accelExpansion);

        PAABB out { { grown.pMin.x, grown.pMin.y, grown.pMin.z },
                    { grown.pMax.x, grown.pMax.y, grown.pMax.z } };
        storePairs(&bvh.leafAABBs[leaf], out);
        LeafTransform lt { { pos.x, pos.y, pos.z }, { rot.w, rot.x, rot.y, rot.z },
                           { scale.d0, scale.d1, scale.d2 } };
        storePairs(&bvh.leafTransforms[leaf], lt);
        bvh.sortedLeaves[leaf] = leaf;
    }
}

// ---- top-down build, one thread per world, only when the world asked for it -----------

__device__ __forceinline__ Vector3 leafCenter(const WorldBVH &bvh, i32 slot)
{
    const PAABB &b = bvh.leafAABBs[bvh.sortedLeaves[slot]];
    Vector3 lo { b.pMin.x, b.pMin.y, b.pMin.z };
    Vector3 hi { b.pMax.x, b.pMax.y, b.pMax.z };
    return (lo + hi) / 2.f;
}

// Partition sortedLeaves[base, base+n) around the midpoint of the centroid
// range on its widest axis; returns the size of the left part (n/2 when the
// partition degenerates).
__device__ i32 midpointPartition(WorldBVH &bvh, i32 base, i32 n)
{
    Vector3 cmin { FLT_MAX, FLT_MAX, FLT_MAX };
    Vector3 cmax { -FLT_MAX, -FLT_MAX, -FLT_MAX };
    for (i32 i = 0; i < n; i++) {
        Vector3 c = leafCenter(bvh, base + i);
        cmin = Vector3::min(cmin, c);
        cmax = Vector3::max(cmax, c);
    }
    Vector3 extent = cmax - cmin;
    int axis;
    if (extent.x > extent.y && extent.x > extent.z) axis = 0;
    else if (extent.y > extent.x && extent.y > extent.z) axis = 1;
    else axis = 2;

    const float split = 0.5f * (cmin[axis] + cmax[axis]);
    i32 lo = 0, hi = n;
    while (lo < hi) {
        while (lo < hi && leafCenter(bvh, base + lo)[axis] < split) ++lo;
        while (lo < hi && leafCenter(bvh, base + hi - 1)[axis] >= split) --hi;
        if (lo < hi) {
            i32 tmp = bvh.sortedLeaves[base + lo];
            bvh.sortedLeaves[base + lo] = bvh.sortedLeaves[base + hi - 1];
            bvh.sortedLeaves[base + hi - 1] = tmp;
            ++lo;
            --hi;
        }
    }
    return (lo > 0 && lo < n) ? lo : n / 2;
}

// Both stacks of the build hold 64 entries, as the reference's (broadphase.cpp:60).  A tree
// too deep for them (clustered leaves make the midpoint splits lopsided) is not built:
// returns false with numTraversal = 0, so no search or query reads a partial leaf list.
constexpr int kRebuildStack = 64;

__device__ bool rebuildWorldBVH(WorldBVH &bvh)
{
    const i32 num_leaves = bvh.numLeaves;
    i32 third = (num_leaves - 1 + 2) / 3;
    bvh.numNodes = (third > 1 ? third : 1) + num_leaves;

    struct Pending {
        i32 node;     // -1 until the entry got its node
        i32 parent;
        i32 offset;
        i32 count;
    };
    Pending stack[kRebuildStack];
    stack[0] = Pending { -1, -1, 0, num_leaves };
    i32 depth = 1;
    i32 next_node = 0;

    while (depth > 0) {
        Pending &top = stack[depth - 1];
        i32 node_id;
        if (top.count <= 4) {
            // leaf-level node: up to four leaves, in sorted order
            node_id = next_node++;
            BVHNode &node = bvh.nodes[node_id];
            node.parentID = top.parent;
            for (int i = 0; i < 4; i++) {
                if (i < top.count) {
                    i32 leaf = bvh.sortedLeaves[top.offset + i];
                    const PAABB box = bvh.leafAABBs[leaf];
                    bvh.leafParents[leaf] = ((u32)node_id << 2) | (u32)i;
                    node.children[i] = (i32)(0x80000000u | (u32)leaf);
                    node.minX[i] = box.pMin.x; node.minY[i] = box.pMin.y; node.minZ[i] = box.pMin.z;
                    node.maxX[i] = box.pMax.x; node.maxY[i] = box.pMax.y; node.maxZ[i] = box.pMax.z;
                } else {
                    node.children[i] = -1;
                    node.minX[i] = FLT_MAX; node.minY[i] = FLT_MAX; node.minZ[i] = FLT_MAX;
                    node.maxX[i] = -FLT_MAX; node.maxY[i] = -FLT_MAX; node.maxZ[i] = -FLT_MAX;
                }
            }
        } else if (top.node == -1) {
            // first visit of an inner entry: take a node, split the range into
            // quarters (half, then each half again) and descend left to right
            if (depth + 4 > kRebuildStack) {
                bvh.numTraversal = 0;
                return false;
            }
            node_id = next_node++;
            top.node = node_id;
            BVHNode &node = bvh.nodes[node_id];
            for (int i = 0; i < 4; i++) node.children[i] = -1;
            node.parentID = top.parent;

            const i32 offset = top.offset, count = top.count;
            const i32 half = midpointPartition(bvh, offset, count);
            const i32 n_left = half, n_right = count - half;
            const i32 q1 = midpointPartition(bvh, offset, n_left);
            const i32 q3 = midpointPartition(bvh, offset + half, n_right);

            stack[depth++] = Pending { -1, node_id, offset + n_left + q3, n_right - q3 };
            stack[depth++] = Pending { -1, node_id, offset + n_left, q3 };
            stack[depth++] = Pending { -1, node_id, offset + q1, n_left - q1 };
            stack[depth++] = Pending { -1, node_id, offset, q1 };
            continue;
        } else {
            node_id = top.node;   // children done
        }

        depth -= 1;
        BVHNode &node = bvh.nodes[node_id];
        if (node.parentID == -1) continue;

        AABB merged = AABB::invalid();
        for (int i = 0; i < 4; i++) {
            if (node.children[i] == -1) break;
            merged = AABB::merge(merged, AABB { { node.minX[i], node.minY[i], node.minZ[i] },
                                                { node.maxX[i], node.maxY[i], node.maxZ[i] } });
        }
        BVHNode &parent = bvh.nodes[node.parentID];
        int slot = 0;
        while (parent.children[slot] != -1) slot++;
        parent.children[slot] = node_id;
        parent.minX[slot] = merged.pMin.x; parent.minY[slot] = merged.pMin.y; parent.minZ[slot] = merged.pMin.z;
        parent.maxX[slot] = merged.pMax.x; parent.maxY[slot] = merged.pMax.y; parent.maxZ[slot] = merged.pMax.z;
    }

    // report order of an un-pruned traversal (include/madrona/broadphase.inl:21-59)
    i32 order_n = 0;
    i32 walk[kRebuildStack];
    walk[0] = 0;
    i32 walk_n = 1;
    while (walk_n > 0) {
        const BVHNode &node = bvh.nodes[walk[--walk_n]];
        for (int i = 0; i < 4; i++) {
            const i32 child = node.children[i];
            if (child == -1) continue;
            if (child & 0x80000000) {
                if (order_n < bvh.numAllocatedLeaves) bvh.traversalOrder[order_n++] = child & 0x7fffffff;
            } else if (walk_n < kRebuildStack) {
                walk[walk_n++] = child;
            } else {
                bvh.numTraversal = 0;
                return false;
            }
        }
    }
    bvh.numTraversal = order_n;
    for (i32 k = 0; k < order_n; k++) {
        const i32 leaf = bvh.traversalOrder[k];
        bvh.leafOrderPos[leaf] = k;
        const u32 packed = bvh.leafParents[leaf];
        const BVHNode &node = bvh.nodes[packed >> 2];
        const int sub = (int)(packed & 3u);
        bvh.orderedBoxes[2 * k] = PVec4 { node.minX[sub], node.minY[sub], node.minZ[sub], node.maxX[sub] };
        bvh.orderedBoxes[2 * k + 1] = PVec4 { node.maxY[sub], node.maxZ[sub], __int_as_float(leaf), 0.f };
    }
    return true;
}

__device__ void refitLeaf(WorldBVH &bvh, i32 leaf);

// Rebuild (rare: after a reset) followed by the refit of every leaf of the
// world, which the fused update+refit kernel skipped for this world.
__device__ __forceinline__ void phaseRebuild(EngineState &S, const PhysicsState &P, const i32 w)
{
    WorldBVH &bvh = worldBVH(S, P, w);
    if (!bvh.forceRebuild) return;
    bvh.forceRebuild = 0;
    if (!rebuildWorldBVH(bvh)) {
        atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);   // the tree is deeper than the build's stacks
        return;
    }
    for (u32 bi = 0; bi < P.numBodyArchetypes; bi++) {
        const BodyArchetype &b = P.bodies[bi];
        const TableDesc &t = S.tables[b.archetype];
        const i32 first_row = t.worldOffsets[w];
        const i32 num_rows = t.worldCounts[w];
        for (i32 row = first_row; row < first_row + num_rows; row++) {
            if (((const i32 *)t.columns[1])[row] != w) continue;
            refitLeaf(bvh, bodyCol<i32>(S, b, PCLeafID, row));
        }
    }
}

// Grow-only refit: push the leaf's box into its slot, then keep growing
// ancestors while something actually grew (broadphase.cpp:550-647).
__device__ void refitLeaf(WorldBVH &bvh, i32 leaf)
{
    const PAABB box = bvh.leafAABBs[leaf];
    const u32 packed = bvh.leafParents[leaf];
    i32 node_idx = (i32)(packed >> 2);
    const int sub = (int)(packed & 3u);
    BVHNode &leaf_node = bvh.nodes[node_idx];
    {
        bool grew = false;
        float prev;
        prev = leaf_node.minX[sub]; if (box.pMin.x < prev) { leaf_node.minX[sub] = box.pMin.x; grew = true; }
        prev = leaf_node.minY[sub]; if (box.pMin.y < prev) { leaf_node.minY[sub] = box.pMin.y; grew = true; }
        prev = leaf_node.minZ[sub]; if (box.pMin.z < prev) { leaf_node.minZ[sub] = box.pMin.z; grew = true; }
        prev = leaf_node.maxX[sub]; if (box.pMax.x > prev) { leaf_node.maxX[sub] = box.pMax.x; grew = true; }
        prev = leaf_node.maxY[sub]; if (box.pMax.y > prev) { leaf_node.maxY[sub] = box.pMax.y; grew = true; }
        prev = leaf_node.maxZ[sub]; if (box.pMax.z > prev) { leaf_node.maxZ[sub] = box.pMax.z; grew = true; }
        if (!grew) return;
        // keep the flat list in step with the slot box (only this leaf's thread writes either)
        const i32 k = bvh.leafOrderPos[leaf];
        float4 *flat = reinterpret_cast<float4 *>(bvh.orderedBoxes);
        flat[2 * k] = make_float4(leaf_node.minX[sub], leaf_node.minY[sub], leaf_node.minZ[sub], leaf_node.maxX[sub]);
        flat[2 * k + 1] = make_float4(leaf_node.maxY[sub], leaf_node.maxZ[sub], __int_as_float(leaf), 0.f);
    }
    i32 child = node_idx;
    node_idx = leaf_node.parentID;
    while (node_idx != -1) {
        BVHNode &node = bvh.nodes[node_idx];
        int slot = -1;
        for (int j = 0; j < 4; j++) {
            if (node.children[j] == child) { slot = j; break; }
        }
        if (slot < 0) return;
        // the six bounds are fetched together (L2: other SMs grow them with atomics), the
        // components that this leaf extends are pushed with fire-and-forget atomics; a bound
        // that a concurrent leaf has grown past ours meanwhile only costs a redundant climb
        const float o0 = __ldcg(&node.minX[slot]), o1 = __ldcg(&node.minY[slot]), o2 = __ldcg(&node.minZ[slot]);
        const float o3 = __ldcg(&node.maxX[slot]), o4 = __ldcg(&node.maxY[slot]), o5 = __ldcg(&node.maxZ[slot]);
        bool grew = false;
        if (box.pMin.x < o0) { atomicMinFloat(&node.minX[slot], box.pMin.x); grew = true; }
        if (box.pMin.y < o1) { atomicMinFloat(&node.minY[slot], box.pMin.y); grew = true; }
        if (box.pMin.z < o2) { atomicMinFloat(&node.minZ[slot], box.pMin.z); grew = true; }
        if (box.pMax.x > o3) { atomicMaxFloat(&node.maxX[slot], box.pMax.x); grew = true; }
        if (box.pMax.y > o4) { atomicMaxFloat(&node.maxY[slot], box.pMax.y); grew = true; }
        if (box.pMax.z > o5) { atomicMaxFloat(&node.maxZ[slot], box.pMax.z); grew = true; }
        if (!grew) break;
        child = node_idx;
        node_idx = node.parentID;
    }
}

__device__ __forceinline__ void rowRefit(const EngineState &S, const PhysicsState &P, const BodyArchetype &b, const i32 row, const i32 w)
{
    refitLeaf(worldBVH(S, P, w), bodyCol<i32>(S, b, PCLeafID, row));
}

// A body takes part in contact ordering unless writing it back is a no-op:
// static (inverse mass / inertia forced to 0, so the solves add exactly +-0 to
// x and q) AND its rotation is a bitwise fixpoint of normalize() AND no
// component of x or q is -0 (-0 + (+0) == +0: two writers of one level would
// store -0 and +0, where the sequential sweep ends at +0).  Decided once per
// step by the candidate search (a fixpoint stays one: the solvers write back
// normalize(q) == q; treating a body that BECAME a fixpoint during the step as
// still mutable only adds ordering edges, never removes one).
__device__ __forceinline__ bool rotationIsNormalizeFixpoint(Quat q)
{
    const Quat n = q.normalize();
    return n.w == q.w && n.x == q.x && n.y == q.y && n.z == q.z;
}

__device__ __forceinline__ bool isNegativeZero(float f) { return __float_as_uint(f) == 0x80000000u; }

__device__ __forceinline__ bool writeBackIsNoOp(Vector3 x, Quat q)
{
    if (isNegativeZero(x.x) || isNegativeZero(x.y) || isNegativeZero(x.z)) return false;
    if (isNegativeZero(q.w) || isNegativeZero(q.x) || isNegativeZero(q.y) || isNegativeZero(q.z)) return false;
    return rotationIsNormalizeFixpoint(q);
}

constexpr u32 kUnknownSlot = 0x7fffu;

// Slot of a body inside its world's body list: archetypes ascending, rows in
// order (-1: not a body archetype).  Contacts carry it (Candidate::slots) and the
// solvers stage bodies by it, so both must use this one formula.
__device__ __forceinline__ i32 worldBodySlot(const EngineState &S, const PhysicsState &P, const i32 w,
                                             const u32 arch, const i32 row)
{
    i32 slot_base = 0;
    for (u32 bi = 0; bi < P.numBodyArchetypes; bi++) {
        const TableDesc &bt = S.tables[P.bodies[bi].archetype];
        if (P.bodies[bi].archetype == arch) return slot_base + (row - bt.worldOffsets[w]);
        slot_base += bt.worldCounts[w];
    }
    return -1;
}

// ---- candidate pairs: one warp per world, CPU iteration order -----------------------------

constexpr int kMaxStagedLeaves = 128;          // bodies per world the candidate search handles
constexpr int kLeafMaskWords = kMaxStagedLeaves / 64;

struct __align__(16) StagedLeaf {
    float box[6];       // the leaf's slot in its parent node (grow-only since the last rebuild)
    i32 entityID;
    u32 arch;
    i32 row;
    u32 prims;          // 0 => stale entity / not a rigid body: never a partner
    u32 primBase;       // ObjectManager::primOffsets[object]
    u32 isStatic;
    u32 slotInfo;       // (world body slot << 1) | mutable  (Candidate::slots)
};

struct CandidateScratch {
    StagedLeaf leaves[kPhysWarps][kMaxStagedLeaves];
};

// Appends candidate i of world w to `list` on the lanes where `take` is set: one atomic
// per warp, the lanes' entries in lane order.
__device__ __forceinline__ void appendPairs(const PairList &list, const bool take, const i32 w, const i32 i,
                                            const int lane)
{
    const unsigned mask = __ballot_sync(0xffffffffu, take);
    if (!mask) return;
    i32 at = 0;
    if (lane == 0) at = atomicAdd(&list.counters->count, __popc(mask));
    at = __shfl_sync(0xffffffffu, at, 0);
    if (take) list.entries[at + __popc(mask & ((1u << lane) - 1u))] = PairEntry { w, i };
}

// The rules of the candidate search.  Two kernels search: one warp per world for worlds of
// up to kMaxStagedLeaves leaves (phaseFindCandidates) and one block per world for larger
// ones (phaseFindCandidatesLarge).  Both describe leaves and bodies, test pairs, write
// candidates and fill the step's work lists through the helpers below and differ only in
// how the work is spread and where the staged leaves live, so both emit the same list.

// (world body slot << 1) | mutable of a body (Candidate::slots)
__device__ __forceinline__ u32 bodySlotInfo(const EngineState &S, const PhysicsState &P, const i32 w,
                                            const u32 arch, const i32 row, const bool is_static)
{
    const i32 slot = worldBodySlot(S, P, w, arch, row);
    bool is_mutable = true;
    if (is_static) {
        is_mutable = !writeBackIsNoOp(cachedCol<Vector3>(arch, PCPosition, row),
                                      cachedCol<Quat>(arch, PCRotation, row));
    }
    const u32 s15 = (slot < 0 || slot >= (i32)kUnknownSlot) ? kUnknownSlot : (u32)slot;
    return (s15 << 1) | (is_mutable ? 1u : 0u);
}

// The k-th leaf the world's tree reports, as a partner
__device__ __forceinline__ StagedLeaf describeLeaf(EngineState &S, const PhysicsState &P, const i32 w,
                                                   const WorldBVH &bvh, const ObjectManager &objs, const i32 k)
{
    const float4 b0 = reinterpret_cast<const float4 *>(bvh.orderedBoxes)[2 * k];
    const float4 b1 = reinterpret_cast<const float4 *>(bvh.orderedBoxes)[2 * k + 1];
    const i32 leaf = __float_as_int(b1.z);
    StagedLeaf sl;
    sl.box[0] = b0.x; sl.box[1] = b0.y; sl.box[2] = b0.z;
    sl.box[3] = b0.w; sl.box[4] = b1.x; sl.box[5] = b1.y;
    const u64 packed = bvh.leafEntities[leaf];
    sl.entityID = (i32)(u32)(packed >> 32);
    const u32 gen = (u32)(packed & 0xFFFFFFFFull);
    sl.arch = 0; sl.row = 0; sl.prims = 0; sl.primBase = 0; sl.isStatic = 0; sl.slotInfo = 0;
    if (sl.entityID >= 0 && sl.entityID < S.entityCapacity) {
        const EntitySlot es = S.entitySlots[sl.entityID];
        const BodyArchetype *bb = es.gen == gen ? bodyOf(P, (u32)es.a) : nullptr;
        if (bb) {
            sl.arch = (u32)es.a;
            sl.row = es.b;
            sl.isStatic = bodyCol<u32>(S, *bb, PCResponseType, es.b) == kRespStatic ? 1u : 0u;
            const i32 obj = bodyCol<i32>(S, *bb, PCObjectID, es.b);
            sl.prims = objs.primCounts[obj];
            sl.primBase = objs.primOffsets[obj];
            sl.slotInfo = bodySlotInfo(S, P, w, sl.arch, sl.row, sl.isStatic != 0);
            if (sl.arch > 0xffu || sl.prims > 0xffu) {
                atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);   // does not fit the packed candidate
                sl.prims = 0;
            }
        }
    }
    return sl;
}

// The iterating body: row `row` of body archetype b (valid: the row is one of world w's)
struct SearchBody {
    i32 id;
    bool isStatic;
    u32 prims;
    u32 primBase;
    u32 info;           // bodySlotInfo
    AABB box;           // its leaf box
};

__device__ __forceinline__ SearchBody describeBody(EngineState &S, const PhysicsState &P, const i32 w,
                                                   const WorldBVH &bvh, const ObjectManager &objs,
                                                   const BodyArchetype &b, const i32 row, const bool valid)
{
    SearchBody sb;
    sb.id = 0;
    sb.isStatic = false;
    sb.prims = 0;
    sb.primBase = 0;
    sb.info = 0;
    sb.box = AABB::invalid();
    if (valid) {
        const TableDesc &t = S.tables[b.archetype];
        const u64 packed = ((const u64 *)t.columns[0])[row];
        sb.id = (i32)(u32)(packed >> 32);
        sb.isStatic = bodyCol<u32>(S, b, PCResponseType, row) == kRespStatic;
        const i32 obj = bodyCol<i32>(S, b, PCObjectID, row);
        sb.prims = objs.primCounts[obj];
        sb.primBase = objs.primOffsets[obj];
        sb.info = bodySlotInfo(S, P, w, b.archetype, row, sb.isStatic);
        if (b.archetype > 0xffu || sb.prims > 0xffu) {
            atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
            sb.prims = 0;
        }
        const PAABB lb = bvh.leafAABBs[bodyCol<i32>(S, b, PCLeafID, row)];
        sb.box = AABB { { lb.pMin.x, lb.pMin.y, lb.pMin.z }, { lb.pMax.x, lb.pMax.y, lb.pMax.z } };
    }
    return sb;
}

// The reference reports the leaf for the body and visits the pair: the body iterates (the
// smaller entity ID) and the two are not both static
__device__ __forceinline__ bool pairsWith(const SearchBody &sb, const bool valid, const StagedLeaf &sl)
{
    const AABB other { { sl.box[0], sl.box[1], sl.box[2] }, { sl.box[3], sl.box[4], sl.box[5] } };
    return valid && sl.prims != 0 && sb.box.overlaps(other) && sb.id < sl.entityID && !(sb.isStatic && sl.isStatic);
}

// Check c of the pair (body, leaf), c in [0, sb.prims * sl.prims): primitive c / sl.prims of
// the body against primitive c % sl.prims of the leaf.
// Resolved once per step: no user node runs inside the physics chain, so ObjectID and the
// primitive tables stay as they are until the last substep.  Order the pair by primitive
// type: sphere(1) < hull(2) < plane(4)
__device__ __forceinline__ Candidate pairCandidate(const ObjectManager &objs, const SearchBody &sb,
                                                   const u32 arch, const i32 row, const StagedLeaf &sl,
                                                   const u32 c)
{
    const u32 a_rel = c / sl.prims, b_rel = c % sl.prims;
    const u32 a_prim = sb.primBase + a_rel, b_prim = sl.primBase + b_rel;
    const u32 ta = objs.prims[a_prim].type, tb = objs.prims[b_prim].type;
    const u32 cls = (ta | tb) << 16;      // the PairClass
    const u32 rel = a_rel | (b_rel << 8) | (ta > tb ? 1u << 16 : 0u);
    return ta > tb
        ? Candidate { b_prim, a_prim, sl.row, row, sl.arch | (arch << 8) | cls,
                      sl.slotInfo | (sb.info << 16), { rel, 0 } }
        : Candidate { a_prim, b_prim, row, sl.row, arch | (sl.arch << 8) | cls,
                      sb.info | (sl.slotInfo << 16), { rel, 0 } };
}

// The step's work lists, hull - hull pairs and the others (one atomic per warp, list and 32
// candidates); with a primitive class table, the pairs of any type that have a hull past the
// staging caps go to a third list instead.  The warp takes the world's candidates
// [first, first + 32), [first + stride, ...) up to `running`, all its lanes together.
__device__ __forceinline__ void appendWorldPairs(const PhysicsState &P, const Candidate *out, const i32 w,
                                                 const i32 running, const i32 first, const i32 stride,
                                                 const int lane)
{
    const unsigned char *const prim_class = P.primClass;     // uniform for the launch
    for (i32 base = first; base < running; base += stride) {
        const i32 i = base + lane;
        bool valid = i < running;
        if (prim_class) {
            bool large = false;
            if (valid) {
                const u32 pa = out[i].aPrim, pb = out[i].bPrim;
                const u32 n = (u32)P.numPrimClasses;
                large = (pa < n ? prim_class[pa] : (u32)PrimTooLarge) != PrimSmall ||
                        (pb < n ? prim_class[pb] : (u32)PrimTooLarge) != PrimSmall;
            }
            appendPairs(P.largePairs, large, w, i, lane);
            valid = valid && !large;
        }
        const bool hh = valid && (out[i].arch >> 16) == PairHullHull;
        appendPairs(P.hullPairs, hh, w, i, lane);
        appendPairs(P.otherPairs, valid && !hh, w, i, lane);
    }
}

// Candidate pairs of one world, in the CPU backend's order (bodies: archetype
// ascending, then row; partners of a body: BVH report order).  The set a
// traversal reports for body a is { leaf b : slotBox(b) overlaps leafBox(a) }
// (ancestor boxes contain their leaves' slot boxes, so pruning removes nothing
// else) and its order is the tree's fixed report order, so the search is a
// uniform loop over the staged leaves instead of 32 divergent stack walks.
// A world of more than kMaxStagedLeaves leaves, up to PhysicsState::maxWorldBodies, goes to
// the large-world list for phaseFindCandidatesLarge instead; past that it raises.
__device__ void phaseFindCandidates(EngineState &S, const PhysicsState &P, const i32 w, const int lane,
                                    const int warp, CandidateScratch &scratch)
{
    const WorldBVH &bvh = worldBVH(S, P, w);
    const ObjectManager &objs = *(const ObjectManager *)bvh.objMgr;
    Candidate *out = P.candidates + (size_t)w * P.maxCandidatesPerWorld;
    StagedLeaf *staged = scratch.leaves[warp];
    i32 running = 0;

    const i32 num_leaves = bvh.numTraversal;
    if (num_leaves > kMaxStagedLeaves) {
        if (lane == 0) {
            if (num_leaves <= P.maxWorldBodies) {
                const i32 at = atomicAdd(&P.largeWorlds.counters->count, 1);
                P.largeWorlds.entries[at] = PairEntry { w, num_leaves };
            } else {
                atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
                P.candCounts[w] = 0;
            }
        }
        return;
    }
    // stage 1: lane k describes the k-th reported leaf
    for (i32 k = lane; k < num_leaves; k += 32) staged[k] = describeLeaf(S, P, w, bvh, objs, k);
    __syncwarp();

    for (u32 bi = 0; bi < P.numBodyArchetypes; bi++) {
        const BodyArchetype &b = P.bodies[bi];
        const TableDesc &t = S.tables[b.archetype];
        const i32 first = t.worldOffsets[w];
        const i32 count = t.worldCounts[w];
        for (i32 base = 0; base < count; base += 32) {
            const i32 row = first + base + lane;
            const bool valid = base + lane < count && ((const i32 *)t.columns[1])[row] == w;
            const SearchBody sb = describeBody(S, P, w, bvh, objs, b, row, valid);

            // stage 2: which staged leaves does this body pair with (bit k of word k / 64)
            unsigned long long partners[kLeafMaskWords];
#pragma unroll
            for (int wd = 0; wd < kLeafMaskWords; wd++) partners[wd] = 0;
            i32 mine = 0;
#pragma unroll
            for (int wd = 0; wd < kLeafMaskWords; wd++) {
                const i32 k_end = min(num_leaves, (wd + 1) * 64);
                for (i32 k = wd * 64; k < k_end; k++) {
                    const StagedLeaf &sl = staged[k];
                    if (pairsWith(sb, valid, sl)) {
                        partners[wd] |= 1ull << (k - wd * 64);
                        mine += (i32)(sb.prims * sl.prims);
                    }
                }
            }
            // exclusive scan across the warp = emission offsets in row order
            i32 incl = mine;
            for (int o = 1; o < 32; o <<= 1) {
                i32 up = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += up;
            }
            const i32 total = __shfl_sync(0xffffffffu, incl, 31);
            i32 at = running + incl - mine;
#pragma unroll
            for (int wd = 0; wd < kLeafMaskWords; wd++) {
                unsigned long long word = partners[wd];
                while (word) {
                    const int k = wd * 64 + __ffsll((long long)word) - 1;
                    word &= word - 1;
                    const StagedLeaf &sl = staged[k];
                    const u32 checks = sb.prims * sl.prims;
                    for (u32 c = 0; c < checks; c++) {
                        if (at < P.maxCandidatesPerWorld) out[at] = pairCandidate(objs, sb, b.archetype, row, sl, c);
                        at++;
                    }
                }
            }
            running += total;
        }
    }
    if (running > P.maxCandidatesPerWorld) {
        if (lane == 0) atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
        running = P.maxCandidatesPerWorld;
    }
    if (lane == 0) P.candCounts[w] = running;

    __syncwarp();
    appendWorldPairs(P, out, w, running, 0, 32, lane);
}

// ---- candidate pairs of worlds past kMaxStagedLeaves leaves: one block per world -----------
// The same flat scan in the same order, spread over a block: thread t describes body
// base + t of the world's body list (archetypes ascending, rows in order), the reported
// leaves are staged kLargeSearchTile at a time in shared memory, a count pass over all
// tiles gives each body its number of checks, a block-wide exclusive scan in body order its
// emission offset, and an emit pass over the tiles writes its candidates in report order.
// Every leaf is tested against every body twice: O(N^2) per world.
constexpr int kLargeSearchThreads = 256;
constexpr int kLargeSearchWarps = kLargeSearchThreads / 32;
constexpr int kLargeSearchTile = 512;

struct LargeSearchScratch {
    StagedLeaf tile[kLargeSearchTile];
    long long warpSums[kLargeSearchWarps];
    i32 ticket;
};

__device__ __forceinline__ void stageLeafTile(EngineState &S, const PhysicsState &P, const i32 w,
                                              const WorldBVH &bvh, const ObjectManager &objs,
                                              LargeSearchScratch &sh, const i32 first, const i32 n)
{
    __syncthreads();      // the previous tile is no longer read
    for (i32 k = threadIdx.x; k < n; k += kLargeSearchThreads) sh.tile[k] = describeLeaf(S, P, w, bvh, objs, first + k);
    __syncthreads();
}

__device__ __forceinline__ void phaseFindCandidatesLarge(EngineState &S, const PhysicsState &P, const i32 w,
                                                         LargeSearchScratch &sh)
{
    const WorldBVH &bvh = worldBVH(S, P, w);
    const ObjectManager &objs = *(const ObjectManager *)bvh.objMgr;
    Candidate *out = P.candidates + (size_t)w * P.maxCandidatesPerWorld;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const i32 num_leaves = bvh.numTraversal;
    const long long max_cands = P.maxCandidatesPerWorld;
    long long running = 0;     // no wrap-around before the cap check, whatever the world holds
    i32 staged_first = -1;     // first leaf of the tile in shared memory

    for (u32 bi = 0; bi < P.numBodyArchetypes; bi++) {
        const BodyArchetype &b = P.bodies[bi];
        const TableDesc &t = S.tables[b.archetype];
        const i32 first = t.worldOffsets[w];
        const i32 count = t.worldCounts[w];
        for (i32 base = 0; base < count; base += kLargeSearchThreads) {
            const i32 row = first + base + tid;
            const bool valid = base + tid < count && ((const i32 *)t.columns[1])[row] == w;
            const SearchBody sb = describeBody(S, P, w, bvh, objs, b, row, valid);

            // count pass
            long long mine = 0;
            for (i32 t0 = 0; t0 < num_leaves; t0 += kLargeSearchTile) {
                const i32 n = min(kLargeSearchTile, num_leaves - t0);
                if (t0 != staged_first) {
                    stageLeafTile(S, P, w, bvh, objs, sh, t0, n);
                    staged_first = t0;
                }
                for (i32 k = 0; k < n; k++) {
                    const StagedLeaf &sl = sh.tile[k];
                    if (pairsWith(sb, valid, sl)) mine += (long long)(sb.prims * sl.prims);
                }
            }
            // exclusive scan over the block = emission offsets in body order
            long long incl = mine;
            for (int o = 1; o < 32; o <<= 1) {
                const long long up = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += up;
            }
            if (lane == 31) sh.warpSums[warp] = incl;
            __syncthreads();
            long long before = 0, total = 0;
            for (int i = 0; i < kLargeSearchWarps; i++) {
                const long long s = sh.warpSums[i];
                if (i < warp) before += s;
                total += s;
            }
            long long at = running + before + incl - mine;

            // emit pass: the tiles again, in report order
            for (i32 t0 = 0; t0 < num_leaves; t0 += kLargeSearchTile) {
                const i32 n = min(kLargeSearchTile, num_leaves - t0);
                if (t0 != staged_first) {
                    stageLeafTile(S, P, w, bvh, objs, sh, t0, n);
                    staged_first = t0;
                }
                for (i32 k = 0; k < n && mine != 0; k++) {
                    const StagedLeaf &sl = sh.tile[k];
                    if (!pairsWith(sb, valid, sl)) continue;
                    const u32 checks = sb.prims * sl.prims;
                    for (u32 c = 0; c < checks && at < max_cands; c++, at++) {
                        out[at] = pairCandidate(objs, sb, b.archetype, row, sl, c);
                    }
                }
            }
            running += total;
            __syncthreads();   // warpSums is read by all before the next body chunk writes it
        }
    }
    if (running > max_cands) {
        if (tid == 0) atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
        running = max_cands;
    }
    if (tid == 0) P.candCounts[w] = (i32)running;

    __syncthreads();   // the block's candidates are written before its warps list them
    appendWorldPairs(P, out, w, (i32)running, warp * 32, kLargeSearchThreads, lane);
}

// =============================================================================================
// Integration (xpbd.cpp:100-185) and velocity update (xpbd.cpp:738-779)
// =============================================================================================

__device__ __forceinline__ void rowIntegrate(const EngineState &S, const PhysicsState &P, const BodyArchetype &b, const i32 row, const i32 w)
{
    {

        Vector3 x = bodyCol<Vector3>(S, b, PCPosition, row);
        Quat q = loadQuat(&bodyCol<Quat>(S, b, PCRotation, row));
        const PVelocity vel = loadPairs(&bodyCol<PVelocity>(S, b, PCVelocity, row));
        Vector3 v = vel.linear;
        Vector3 omega = vel.angular;
        const u32 resp = bodyCol<u32>(S, b, PCResponseType, row);

        PPosRot &prev = bodyCol<PPosRot>(S, b, PCPrevState, row);
        PPosRot &pre_pos = bodyCol<PPosRot>(S, b, PCPreSolvePos, row);
        PVelocity &pre_vel = bodyCol<PVelocity>(S, b, PCPreSolveVel, row);

        prev.x = x;
        prev.q = q;
        if (resp == kRespStatic) {
            pre_pos.x = x;
            pre_pos.q = q;
            storePairs(&pre_vel, PVelocity { Vector3::zero(), Vector3::zero() });
            return;
        }

        const PhysicsWorldParams &params = worldParams(S, P, w);
        const ObjectManager &objs = worldObjects(S, P, w);
        const RigidBodyMetadata &meta = objs.metadata[bodyCol<i32>(S, b, PCObjectID, row)];
        const float inv_m = meta.invMass;
        const Vector3 inv_I = meta.invInertia;
        const float h = params.h;
        const Vector3 g { params.g.x, params.g.y, params.g.z };
        const Vector3 ext_force = bodyCol<Vector3>(S, b, PCExtForce, row);
        const Vector3 ext_torque = bodyCol<Vector3>(S, b, PCExtTorque, row);

        if (resp == kRespDynamic) v += h * g;
        v += h * inv_m * ext_force;
        x += h * v;

        const Vector3 I { inv_I.x == 0 ? 0.0f : 1.0f / inv_I.x,
                          inv_I.y == 0 ? 0.0f : 1.0f / inv_I.y,
                          inv_I.z == 0 ? 0.0f : 1.0f / inv_I.z };
        const Quat to_local = q.inv();
        const Vector3 tau_local = to_local.rotateVec(ext_torque);
        Vector3 omega_local = to_local.rotateVec(omega);
        const Vector3 I_omega = mulDiag(I, omega_local);
        // Euler's equations in the body frame (gyroscopic term included)
        omega_local += h * mulDiag(inv_I, tau_local - cross(omega_local, I_omega));
        omega = q.rotateVec(omega_local);

        const Quat spin = Quat::fromAngularVec(0.5f * h * omega);
        q += spin * q;
        q = q.normalize();

        bodyCol<Vector3>(S, b, PCPosition, row) = x;
        storeQuat(&bodyCol<Quat>(S, b, PCRotation, row), q);
        pre_pos.x = x;
        pre_pos.q = q;
        storePairs(&pre_vel, PVelocity { v, omega });
    }
}

// ---- TGS (src/physics/tgs.cpp): the reference's solver skeleton integrates and nothing else
__device__ __forceinline__ void rowTGSVelocities(const EngineState &S, const PhysicsState &P, const BodyArchetype &b, const i32 row, const i32 w)
{
    const u32 resp = bodyCol<u32>(S, b, PCResponseType, row);
    if (resp == kRespStatic) return;
    PVelocity &vel_ref = bodyCol<PVelocity>(S, b, PCVelocity, row);
    const PVelocity vel = loadPairs(&vel_ref);
    Vector3 v = vel.linear;
    Vector3 omega = vel.angular;
    const Quat q = loadQuat(&bodyCol<Quat>(S, b, PCRotation, row));
    const PhysicsWorldParams &params = worldParams(S, P, w);
    const ObjectManager &objs = worldObjects(S, P, w);
    const RigidBodyMetadata &meta = objs.metadata[bodyCol<i32>(S, b, PCObjectID, row)];
    const float inv_m = meta.invMass;
    const Vector3 inv_I = meta.invInertia;
    const float h = params.h;
    const Vector3 g { params.g.x, params.g.y, params.g.z };
    if (resp == kRespDynamic) v += h * g;
    v += h * inv_m * bodyCol<Vector3>(S, b, PCExtForce, row);
    const Vector3 I { inv_I.x == 0 ? 0.0f : 1.0f / inv_I.x,
                      inv_I.y == 0 ? 0.0f : 1.0f / inv_I.y,
                      inv_I.z == 0 ? 0.0f : 1.0f / inv_I.z };
    const Quat to_local = q.inv();
    const Vector3 tau_local = to_local.rotateVec(bodyCol<Vector3>(S, b, PCExtTorque, row));
    Vector3 omega_local = to_local.rotateVec(omega);
    // NB: the reference multiplies I by the WORLD-space omega here (tgs.cpp:133-134)
    omega_local += h * mulDiag(inv_I, tau_local - cross(omega_local, mulDiag(I, omega)));
    omega = q.rotateVec(omega_local);
    storePairs(&vel_ref, PVelocity { v, omega });
}

__device__ __forceinline__ void rowTGSPositions(const EngineState &S, const PhysicsState &P, const BodyArchetype &b, const i32 row, const i32 w)
{
    const float h = worldParams(S, P, w).h;
    Vector3 x = bodyCol<Vector3>(S, b, PCPosition, row);
    Quat q = loadQuat(&bodyCol<Quat>(S, b, PCRotation, row));
    const PVelocity vel = loadPairs(&bodyCol<PVelocity>(S, b, PCVelocity, row));
    x += h * vel.linear;
    const Quat spin = Quat::fromAngularVec(0.5f * h * vel.angular);
    q += spin * q;
    q = q.normalize();
    bodyCol<Vector3>(S, b, PCPosition, row) = x;
    storeQuat(&bodyCol<Quat>(S, b, PCRotation, row), q);
}

__device__ __forceinline__ void rowSetVelocity(const EngineState &S, const PhysicsState &P, const BodyArchetype &b, const i32 row, const i32 w)
{
    {
        const float h = worldParams(S, P, w).h;
        const Vector3 x = bodyCol<Vector3>(S, b, PCPosition, row);
        const Quat q = loadQuat(&bodyCol<Quat>(S, b, PCRotation, row));
        const PPosRot prev = bodyCol<PPosRot>(S, b, PCPrevState, row);

        // bitwise-equal orientations mean exactly zero angular velocity
        Quat dq;
        if (q.w != prev.q.w || q.x != prev.q.x || q.y != prev.q.y || q.z != prev.q.z) {
            dq = q * prev.q.inv();
        } else {
            dq = Quat { 1, 0, 0, 0 };
        }
        const Vector3 new_omega = 2.f / h * Vector3 { dq.x, dq.y, dq.z };

        PVelocity out;
        out.linear = (x - prev.x) / h;
        out.angular = dq.w > 0.f ? new_omega : -new_omega;
        storePairs(&bodyCol<PVelocity>(S, b, PCVelocity, row), out);
    }
}

// =============================================================================================
// Narrowphase (scalar SAT path of the reference)
// =============================================================================================

// Every pair is worked on by a GROUP of lanes (the pair's setup is loaded by each
// lane, the same addresses): the vertex / face / edge scans, the polygon filter and
// the manifold reduction are spread over the group, and every sequential "first
// strictly better" scan of the reference becomes a reduction that keeps the lowest
// index among the best -- order independent, so bit-identical.  Hull - hull pairs
// take kGroupLanes lanes (4 pairs per warp); the cheaper hull - plane pairs take
// kPlaneLanes (see physNarrowphaseKernel).
constexpr int kGroupLanes = 8;
constexpr int kClipCap = kMaxFaceVerts * 2 + 4;

__device__ __forceinline__ float planeDistance(const Plane &pl, Vector3 p)
{
    return dot(p, pl.normal) - pl.d;
}

__device__ __forceinline__ bool gaussMapArcsCross(Vector3 a, Vector3 b, Vector3 c, Vector3 d)
{
    Vector3 bxa = b.cross(a);
    Vector3 dxc = d.cross(c);
    float cba = c.dot(bxa);
    float dba = d.dot(bxa);
    float adc = a.dot(dxc);
    float bdc = b.dot(dxc);
    return cba * dba < 0.0f && adc * bdc < 0.0f && cba * bdc > 0.0f;
}

// Sutherland-Hodgman against one plane; "<= 0" is inside (narrowphase.cpp:617-652).
// dst holds `cap` points: returns -1, having written nothing past dst[cap - 1], when
// the clipped polygon would not fit.
__device__ __forceinline__ int clipAgainst(Vector3 *dst, const Plane &pl, const Vector3 *src, int n, int cap)
{
    int m = 0;
    Vector3 v1 = src[n - 1];
    float d1 = planeDistance(pl, v1);
#pragma unroll 1
    for (int i = 0; i < n; i++) {
        Vector3 v2 = src[i];
        float d2 = planeDistance(pl, v2);
        if (d1 <= 0.0f && d2 <= 0.0f) {
            if (m == cap) return -1;
            dst[m++] = v2;
        } else if (d1 <= 0.0f && d2 > 0.0f) {
            if (m == cap) return -1;
            dst[m++] = v1 + (v2 - v1) * (-d1 / pl.normal.dot(v2 - v1));
        } else if (d2 <= 0.0f && d1 > 0.0f) {
            if (m + 2 > cap) return -1;
            dst[m++] = v1 + (v2 - v1) * (-d1 / pl.normal.dot(v2 - v1));
            dst[m++] = v2;
        }
        v1 = v2;
        d1 = d2;
    }
    return m;
}

// closest points of two segments, clamped (narrowphase.cpp:1037-1071); only the
// point on segment 1 is used by the caller
__device__ Vector3 closestOnFirstSegment(Vector3 p1, Vector3 q1, Vector3 p2, Vector3 q2)
{
    Vector3 v1 = q1 - p1;
    Vector3 v2 = q2 - p2;
    Vector3 v21 = p2 - p1;
    float d22 = v2.dot(v2);
    float d11 = v1.dot(v1);
    float d21 = v2.dot(v1);
    float d211 = v21.dot(v1);
    float d212 = v21.dot(v2);
    float denom = d21 * d21 - d22 * d11;
    float s;
    if (fabsf(denom) < 0.00001f) {
        s = 0.0f;
    } else {
        s = (d212 * d21 - d22 * d211) / denom;
    }
    s = fmaxf(fminf(s, 1.0f), 0.0f);
    return p1 + s * v1;
}

// Contacts are written field by field straight into their slot (no staging copy).
__device__ __forceinline__ void writeContactHeader(Contact &c, u32 ref_arch, i32 ref_row, u32 ref_info,
                                                   u32 alt_arch, i32 alt_row, u32 alt_info, int count,
                                                   Vector3 normal)
{
    c.refArch = ref_arch; c.refRow = ref_row;
    c.altArch = alt_arch; c.altRow = alt_row;
    c.numPoints = count;
    c.normal = PVec3 { normal.x, normal.y, normal.z };
    c.lambdaN = 0.f;
    c.refInfo = ref_info;
    c.altInfo = alt_info;
    c.level = 0;
}

__device__ __forceinline__ void writeContactPoint(Contact &c, int i, Vector3 p, float depth)
{
    c.points[i][0] = p.x;
    c.points[i][1] = p.y;
    c.points[i][2] = p.z;
    c.points[i][3] = depth;
}

// one lane: a one-point contact, unused points zero
__device__ __forceinline__ void writeSinglePointContact(Contact &c, u32 ref_arch, i32 ref_row, u32 ref_info,
                                                        u32 alt_arch, i32 alt_row, u32 alt_info,
                                                        Vector3 p, Vector3 normal, float depth)
{
    writeContactHeader(c, ref_arch, ref_row, ref_info, alt_arch, alt_row, alt_info, 1, normal);
    writeContactPoint(c, 0, p, depth);
    for (int i = 1; i < 4; i++) writeContactPoint(c, i, Vector3::zero(), 0.f);
}

// ---- one candidate -> at most one contact (narrowphase.cpp:1682-1899 + 1516-1680) ------

// What a pair needs every substep.  Everything fixed for the step (primitives in type
// order, rows, slot infos, pair class) comes resolved in the Candidate.
struct PairSetup {
    u32 aArch, bArch;
    i32 aRow, bRow;
    u32 aInfo, bInfo;  // (world body slot << 1) | mutable, see Candidate::slots
    const CollisionPrimitive *aPrim, *bPrim;
    Vector3 aPos, bPos;
    Quat aRot, bRot;
    Diag3x3 aScale, bScale;
    u32 test;          // the pair class, 0 = rejected by the primitive boxes
};

__device__ __forceinline__ PairSetup setupPair(const ObjectManager &objs, const Candidate &cand)
{
    PairSetup ps;
    ps.aArch = cand.arch & 0xffu; ps.bArch = (cand.arch >> 8) & 0xffu;
    ps.aRow = cand.aRow; ps.bRow = cand.bRow;
    ps.aInfo = cand.slots & 0xffffu; ps.bInfo = cand.slots >> 16;
    ps.aPrim = &objs.prims[cand.aPrim];
    ps.bPrim = &objs.prims[cand.bPrim];
    ps.aPos = cachedCol<Vector3>(ps.aArch, PCPosition, ps.aRow);
    ps.bPos = cachedCol<Vector3>(ps.bArch, PCPosition, ps.bRow);
    ps.aRot = cachedCol<Quat>(ps.aArch, PCRotation, ps.aRow);
    ps.bRot = cachedCol<Quat>(ps.bArch, PCRotation, ps.bRow);
    ps.aScale = cachedCol<Diag3x3>(ps.aArch, PCScale, ps.aRow);
    ps.bScale = cachedCol<Diag3x3>(ps.bArch, PCScale, ps.bRow);
    AABB a_box = objs.primAABBs[cand.aPrim].applyTRS(ps.aPos, ps.aRot, ps.aScale);
    AABB b_box = objs.primAABBs[cand.bPrim].applyTRS(ps.bPos, ps.bRot, ps.bScale);
    ps.test = a_box.intersects(b_box) ? (cand.arch >> 16) : 0u;
    return ps;
}

struct HullScratch {
    Vector3 verts[2 * kMaxHullVerts];
    Plane planes[2 * kMaxHullFaces];
    Vector3 clipA[kClipCap];
    Vector3 clipB[kClipCap];
    float depths[kClipCap];
};

// Where the group of a hull - hull pair stages both hulls, the clipped polygon and its
// depths, and how much fits: the HullScratch of an 8-lane group, or a warp's slice of
// dynamic shared memory sized from PhysicsState::maxHullSize (physNarrowphaseLargeKernel).
struct HullStage {
    Vector3 *vertsA, *vertsB;
    Plane *planesA, *planesB;
    Vector3 *clipA, *clipB;     // clipCap points each
    float *depths;              // clipCap
    int maxVerts, maxFaces, maxFaceVerts, clipCap;
};

__device__ __forceinline__ HullStage smallHullStage(HullScratch &s)
{
    return HullStage { s.verts, s.verts + kMaxHullVerts, s.planes, s.planes + kMaxHullFaces,
                       s.clipA, s.clipB, s.depths, kMaxHullVerts, kMaxHullFaces, kMaxFaceVerts, kClipCap };
}

// hull - plane pairs: the incident face's points and what groupManifold keeps of them
struct PlaneScratch {
    Vector3 pts[kMaxFaceVerts];
    Vector3 kept[kMaxFaceVerts];
    float depths[kMaxFaceVerts];
    static constexpr int cap = kMaxFaceVerts;
};

// the same in a warp's slice of dynamic shared memory (physNarrowphaseLargeKernel)
struct LargePlaneStage {
    Vector3 *pts, *kept;
    float *depths;
    int cap;
};

// (value, index) of the element a sequential scan would have kept.
struct Winner {
    float sep;
    i32 idx;
};

// Reduction over the lanes of one group (mask gm, xor distances stay inside the
// aligned group).  Input per lane: its own candidate (sep, idx) chosen by the
// same rule over the elements it looked at, or have = false.
// Rule == the scalar loop "keep strictly greater, stop at the first positive":
// lowest index among positives, else lowest index among maxima -- for any number of lanes
// G the elements were dealt to.
template <int G = kGroupLanes>
__device__ __forceinline__ Winner groupSequentialWinner(unsigned gm, float sep, i32 idx, bool have)
{
    const bool positive = have && sep > 0.f;
    if (__any_sync(gm, positive)) {
        i32 cand = positive ? idx : 0x7fffffff;
#pragma unroll
        for (int o = G / 2; o >= 1; o >>= 1) {
            const i32 other = __shfl_xor_sync(gm, cand, o);
            if (other < cand) cand = other;
        }
        const unsigned owner = __ballot_sync(gm, positive && idx == cand);
        const int src = __ffs(owner) - 1;
        return Winner { __shfl_sync(gm, sep, src), cand };
    }
    float s = have ? sep : -FLT_MAX;
    i32 k = have ? idx : 0x7fffffff;
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) {
        const float os = __shfl_xor_sync(gm, s, o);
        const i32 ok = __shfl_xor_sync(gm, k, o);
        if (os > s || (os == s && ok < k)) {
            s = os;
            k = ok;
        }
    }
    return Winner { s, k };
}

// The scalar loop "keep the first strictly smaller (LESS) / greater value than the
// best so far" over the group: every lane passes the first best of the elements it
// looked at (have = false: none beat the loop's start value); the result is the
// lowest index among the best values, idx = 0x7fffffff when no lane has one.
template <bool LESS, int G = kGroupLanes>
__device__ __forceinline__ Winner groupFirstBest(unsigned gm, float v, i32 idx, bool have)
{
    float s = have ? v : (LESS ? FLT_MAX : -FLT_MAX);
    i32 k = have ? idx : 0x7fffffff;
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) {
        const float os = __shfl_xor_sync(gm, s, o);
        const i32 ok = __shfl_xor_sync(gm, k, o);
        if ((LESS ? os < s : os > s) || (os == s && ok < k)) {
            s = os;
            k = ok;
        }
    }
    return Winner { s, k };
}

// face of a hull most anti-parallel to the reference normal, first minimum wins
template <int G = kGroupLanes>
__device__ __forceinline__ i32 groupMostOpposedFace(unsigned gm, int sub, const Plane *planes, u32 num_faces,
                                                    Vector3 ref_normal)
{
    float lowest = FLT_MAX;
    i32 face = 0;
    bool have = false;
    for (u32 f = (u32)sub; f < num_faces; f += G) {
        const float d = dot(planes[f].normal, ref_normal);
        if (d < lowest) {
            lowest = d;
            face = (i32)f;
            have = true;
        }
    }
    return groupFirstBest<true, G>(gm, lowest, face, have).idx;
}

// Keep the points pts[0, n) at or below the reference plane, projected onto it with
// depth = -distance, in order (ballot compaction into kept / depths), then reduce
// them to at most 4 (narrowphase.cpp:771-879): <= 4 pass through, else A (first),
// B (farthest from A), C (largest |area| with AB), Q (most negative area outside
// ABC).  World offset / frame are identity in the only live call sites.  Lanes 0-3
// of the group write points 0-3 of `out`; returns the point count on every lane
// (0: no contact, and nothing was written).
template <int G>
__device__ int groupManifold(unsigned gm, int sub, const Plane &ref_plane, const Vector3 *pts, int n,
                             Vector3 *kept, float *depths, Contact &out)
{
    const unsigned below = (1u << (threadIdx.x & 31)) - 1u;
    int count = 0;
    for (int i0 = 0; i0 < n; i0 += G) {
        const int i = i0 + sub;
        Vector3 p = Vector3::zero();
        float d = 0.f;
        bool keep = false;
        if (i < n) {
            p = pts[i];
            d = planeDistance(ref_plane, p);
            keep = d <= 0.0f;
        }
        const unsigned m = __ballot_sync(gm, keep);
        if (keep) {
            const int at = count + __popc(m & below);
            kept[at] = p - d * ref_plane.normal;
            depths[at] = -d;
        }
        count += __popc(m);
    }
    __syncwarp(gm);
    if (count <= 4) {
        if (count > 0) {
            for (int k = sub; k < 4; k += G) {
                writeContactPoint(out, k, k < count ? kept[k] : Vector3::zero(), k < count ? depths[k] : 0.f);
            }
        }
        return count;
    }
    const Vector3 normal = ref_plane.normal;
    const Vector3 pa = kept[0];

    float far2 = 0.f;                       // B: first strictly farther than 0
    i32 b_idx = 0;
    bool have = false;
    for (int i = 1 + sub; i < count; i += G) {
        const float d2 = pa.distance2(kept[i]);
        if (d2 > far2) {
            far2 = d2;
            b_idx = i;
            have = true;
        }
    }
    b_idx = groupFirstBest<false, G>(gm, far2, b_idx, have).idx;
    if (b_idx == 0x7fffffff) return 0;
    const Vector3 pb = kept[b_idx];
    const Vector3 ba = pb - pa;

    float best_area = 0.f;                  // C: first strictly larger |area| than 0
    i32 c_idx = 0;
    have = false;
    for (int i = 1 + sub; i < count; i += G) {
        Vector3 bc = kept[i] - pb;
        float signed_area = normal.dot(cross(ba, bc));
        float area = copysignf(signed_area, 1.f);
        if (area > best_area) {
            best_area = area;
            c_idx = i;
            have = true;
        }
    }
    // NB: the reference stores the winning area's sign in a bool, so its
    // "sign == -1" winding flip never fires; there is nothing to reproduce.
    c_idx = groupFirstBest<false, G>(gm, best_area, c_idx, have).idx;
    if (c_idx == 0x7fffffff) return 0;
    const Vector3 pc = kept[c_idx];

    Vector3 cb = pc - pb;
    Vector3 ac = pa - pc;
    float most_neg = 0.f;                   // Q: first strictly more negative than 0
    i32 q_idx = 0;
    have = false;
    for (int i = 1 + sub; i < count; i += G) {
        Vector3 aq = pa - kept[i];
        Vector3 qc = kept[i] - pc;
        float abq = normal.dot(cross(ba, aq));
        float bcq = normal.dot(cross(cb, qc));
        float caq = normal.dot(cross(aq, ac));
        float lowest = fminf(abq, fminf(bcq, caq));
        if (lowest < most_neg) {
            most_neg = lowest;
            q_idx = i;
            have = true;
        }
    }
    q_idx = groupFirstBest<true, G>(gm, most_neg, q_idx, have).idx;
    if (q_idx == 0x7fffffff) return 0;
    for (int k = sub; k < 4; k += G) {
        const i32 src = k == 0 ? 0 : k == 1 ? b_idx : k == 2 ? c_idx : q_idx;
        writeContactPoint(out, k, kept[src], depths[src]);
    }
    return 4;
}

struct SphereHullResult {
    Vector3 point;
    Vector3 normal;
    float depth;
    i32 hit;          // 1 contact, 0 none, -1 hull too large for the staging array
};

// sphere (a) - hull (b) by the G lanes of a group: GJK closest point of the hull to the
// sphere centre on the group's first lane, SAT over the face planes when the centre is
// inside, the faces dealt to the lanes (narrowphase.cpp:1326-1402).  The lanes stage the
// placed vertices in `verts`, which the caller checked the hull against.  `hit` is the
// same on every lane; point, normal and depth are set on the group's first lane.
template <int G>
__device__ __forceinline__ SphereHullResult sphereHullGroup(Vector3 a_pos, float radius, Vector3 b_pos, Quat b_rot,
                                                            Diag3x3 b_scale, const HalfEdgeMesh &bm, Vector3 *verts,
                                                            const unsigned gm, const int sub)
{
    SphereHullResult res { Vector3::zero(), Vector3::zero(), 0.f, 0 };
    // the hull relative to the sphere centre, so the query point is the origin
    const Vector3 hull_origin = b_pos - a_pos;
    const Mat3x3 rot = Mat3x3::fromQuat(b_rot);
    const Mat3x3 vert_m = rot * b_scale;
    const Mat3x3 norm_m = rot * b_scale.inv();
#pragma unroll 1
    for (u32 i = (u32)sub; i < bm.numVertices; i += G) verts[i] = vert_m * bm.vertices[i] + hull_origin;
    if constexpr (G > 1) __syncwarp(gm);

    Vector3 to_hull = Vector3::zero();
    float dist2 = 0.f;
    if (sub == 0) dist2 = madrona::geo::hullVerticesClosestPointToOriginGJK(verts, bm.numVertices, 1e-10f, &to_hull);
    if constexpr (G > 1) dist2 = __shfl_sync(gm, dist2, __ffs(gm) - 1);
    if (dist2 > radius * radius) return res;

    if (dist2 == 0.f) {
        // centre inside the hull: least-penetrated face, the first maximum of the face scan
        float best = -FLT_MAX;
        i32 best_face = 0;
        Vector3 best_n = Vector3::zero();
        bool have = false;
#pragma unroll 1
        for (u32 f = (u32)sub; f < bm.numFaces; f += G) {
            const Plane local = bm.facePlanes[f];
            const Vector3 on_plane = vert_m * (local.normal * local.d) + hull_origin;
            const Vector3 n = (norm_m * local.normal).normalize();
            const float face_dist = -dot(n, on_plane);
            if (face_dist > best) {
                best = face_dist;
                best_face = (i32)f;
                best_n = n;
                have = true;
            }
        }
        const Winner win = groupFirstBest<false, G>(gm, best, best_face, have);
        // no face beat the scan's start value: it keeps -FLT_MAX and a zero normal
        const bool found = win.idx != 0x7fffffff;
        const float max_sep = found ? win.sep : -FLT_MAX;
        if (max_sep > 0.f) return res;      // GJK and SAT disagree by rounding
        Vector3 sep_normal = best_n;
        if constexpr (G > 1) {
            // the winning lane's normal to the group's first lane
            const unsigned owner = __ballot_sync(gm, have && best_face == win.idx);
            const int src = owner ? __ffs(owner) - 1 : __ffs(gm) - 1;
            sep_normal.x = __shfl_sync(gm, best_n.x, src);
            sep_normal.y = __shfl_sync(gm, best_n.y, src);
            sep_normal.z = __shfl_sync(gm, best_n.z, src);
        }
        res.point = a_pos + sep_normal * radius;
        res.normal = sep_normal;
        res.depth = -max_sep;
    } else {
        const float to_hull_len = sqrtf(dist2);
        const Vector3 normal = to_hull / to_hull_len;
        res.point = a_pos + normal * radius;
        res.normal = -normal;
        res.depth = radius - to_hull_len;
    }
    res.hit = 1;
    return res;
}

// One lane of physNarrowphaseKernel, the vertices in a per-thread array.  Out of line and
// by value: rare in the box-world fixtures, and inlining the GJK loop doubles the
// narrowphase kernel's code size.
__device__ __noinline__ SphereHullResult sphereHullContact(Vector3 a_pos, float radius, Vector3 b_pos,
                                                           Quat b_rot, Diag3x3 b_scale,
                                                           const HalfEdgeMesh *mesh)
{
    if (mesh->numVertices > (u32)kMaxHullVerts) return SphereHullResult { Vector3::zero(), Vector3::zero(), 0.f, -1 };
    Vector3 verts[kMaxHullVerts];
    return sphereHullGroup<1>(a_pos, radius, b_pos, b_rot, b_scale, *mesh, verts, 1u << (threadIdx.x & 31), 0);
}

// sphere - sphere, sphere - plane, sphere - hull: one lane of the group.
// Single-point contacts store (ref, alt) = (b, a).
template <bool SPHERE_HULL>
__device__ bool singlePointPair(EngineState &S, const PairSetup &ps, Contact &out)
{
    switch (ps.test) {
    case PairSphereSphere: {
        const float ra = ps.aScale.d0 * ps.aPrim->sphereRadius;
        const float rb = ps.bScale.d0 * ps.bPrim->sphereRadius;
        const Vector3 to_b = ps.bPos - ps.aPos;
        const float dist = to_b.length();
        if (dist > ra + rb) return false;
        const Vector3 n = dist > 0.f ? to_b / dist : madrona::math::up;
        writeSinglePointContact(out, ps.bArch, ps.bRow, ps.bInfo, ps.aArch, ps.aRow, ps.aInfo,
                                ps.aPos + ra * n, n, ra + rb - dist);
        return true;
    }
    case PairSpherePlane: {
        const float ra = ps.aScale.d0 * ps.aPrim->sphereRadius;
        const Vector3 n = ps.bRot.rotateVec(Vector3 { 0, 0, 1 });
        const float d = n.dot(ps.bPos);
        const float t = n.dot(ps.aPos) - d;
        const float pen = ra - t;
        if (pen < 0) return false;
        writeSinglePointContact(out, ps.bArch, ps.bRow, ps.bInfo, ps.aArch, ps.aRow, ps.aInfo,
                                ps.aPos - t * n, n, pen);
        return true;
    }
    case PairSphereHull: {
        if constexpr (SPHERE_HULL) {
            const SphereHullResult r = sphereHullContact(ps.aPos, ps.aScale.d0 * ps.aPrim->sphereRadius,
                                                         ps.bPos, ps.bRot, ps.bScale, &ps.bPrim->hull);
            if (r.hit < 0) atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
            if (r.hit <= 0) return false;
            writeSinglePointContact(out, ps.bArch, ps.bRow, ps.bInfo, ps.aArch, ps.aRow, ps.aInfo,
                                    r.point, r.normal, r.depth);
            return true;
        } else {
            // a sphere appeared after the launch graph was built without the
            // sphere-hull path: rebuild the launch graph
            atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
            return false;
        }
    }
    default:
        atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
        return false;
    }
}

// hull (a) - plane (b, the reference).  The hull is never stored: each lane places
// the vertices and face normals it reads (vertex = R S v + t, normal =
// normalize(R S^-1 n)).  Returns, on every lane of the group, whether a contact
// was written to `out`.  Stage: PlaneScratch or LargePlaneStage.
template <int G, typename Stage>
__device__ bool hullPlaneGroup(EngineState &S, const PairSetup &ps, Stage &scratch, const unsigned gm,
                               const int sub, Contact &out)
{
    const HalfEdgeMesh &am = ps.aPrim->hull;
    const Mat3x3 rot = Mat3x3::fromQuat(ps.aRot);
    const Mat3x3 vert_m = rot * ps.aScale;
    const Mat3x3 norm_m = rot * ps.aScale.inv();
    const Vector3 n = ps.bRot.rotateVec(Vector3 { 0, 0, 1 });
    const Plane plane { n, dot(n, ps.bPos) };

    float lowest = FLT_MAX;                 // support distance: a minimum, in any order
    for (u32 i = (u32)sub; i < am.numVertices; i += G) {
        const Vector3 p = vert_m * am.vertices[i] + ps.aPos;
        const float along = dot(p, plane.normal);
        if (along < lowest) lowest = along;
    }
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) {
        const float other = __shfl_xor_sync(gm, lowest, o);
        if (other < lowest) lowest = other;
    }
    if (lowest - plane.d > 0.0f) return false;

    float most = FLT_MAX;                   // most opposed face, first minimum
    i32 face = 0;
    bool have = false;
    for (u32 f = (u32)sub; f < am.numFaces; f += G) {
        const Vector3 face_n = (norm_m * am.facePlanes[f].normal).normalize();
        const float d = dot(face_n, plane.normal);
        if (d < most) {
            most = d;
            face = (i32)f;
            have = true;
        }
    }
    const i32 inc_face = groupFirstBest<true, G>(gm, most, face, have).idx;
    if (inc_face == 0x7fffffff) return false;

    // incident-face points, point k on lane k % G
    int nv = 0;
    u32 he = am.faceBaseHalfEdges[inc_face];
    const u32 start = he;
    do {
        const HalfEdge cur = am.halfEdges[he];
        he = cur.next;
        if (nv < scratch.cap && nv % G == sub) scratch.pts[nv] = vert_m * am.vertices[cur.rootVertex] + ps.aPos;
        nv++;
    } while (he != start && nv <= scratch.cap);
    if (nv > scratch.cap) {
        if (sub == 0) atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
        return false;
    }
    __syncwarp(gm);
    const int count = groupManifold<G>(gm, sub, plane, scratch.pts, nv, scratch.kept, scratch.depths, out);
    if (count == 0) return false;
    if (sub == 0) writeContactHeader(out, ps.bArch, ps.bRow, ps.bInfo, ps.aArch, ps.aRow, ps.aInfo, count, plane.normal);
    return true;
}

// faces of one hull against the other hull's vertices: lane `sub` measures faces
// sub, sub + G, ... in ascending order with the scalar rule, then the group combines
// (narrowphase.cpp:339-365)
template <int G = kGroupLanes>
__device__ __forceinline__ Winner groupFaceQuery(unsigned gm, int sub, const Plane *planes, u32 num_faces,
                                                 const Vector3 *other_verts, u32 other_num_verts)
{
    float best = -FLT_MAX;
    i32 best_face = 0x7fffffff;
    bool have = false;
    for (u32 f = (u32)sub; f < num_faces; f += G) {
        const Plane pl = planes[f];
        float lowest = FLT_MAX;
#pragma unroll 1
        for (u32 i = 0; i < other_num_verts; i++) {
            float along = dot(other_verts[i], pl.normal);
            if (along < lowest) lowest = along;
        }
        const float sep = lowest - pl.d;
        if (!have || sep > best) {
            // first element, or strictly greater than what this lane kept so far
            best = sep;
            best_face = (i32)f;
            have = true;
            if (sep > 0.f) break;    // the scalar loop stops at the first positive
        }
    }
    return groupSequentialWinner<G>(gm, best, best_face, have);
}

// Executed by the G lanes of one group for the hull - hull pair `ps` (every lane
// holds the same copy), staging in `st`.  Returns, on every lane of the group, whether
// a contact was written to `out`.
template <int G>
__device__ bool hullHullGroup(EngineState &S, const PairSetup &ps, const HullStage &st, const unsigned gm,
                              const int sub, Contact &out)
{
    const HalfEdgeMesh &am = ps.aPrim->hull;
    const HalfEdgeMesh &bm = ps.bPrim->hull;
    const u32 nva = am.numVertices, nvb = bm.numVertices, nfa = am.numFaces, nfb = bm.numFaces;
    if (nva > (u32)st.maxVerts || nvb > (u32)st.maxVerts ||
            nfa > (u32)st.maxFaces || nfb > (u32)st.maxFaces) {
        if (sub == 0) atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
        return false;
    }

    // -- both hulls into shared memory (vertex = R S v + t, plane via R S^-1,
    // plane offset through a transformed point of the plane: narrowphase.cpp:151-223)
    Vector3 *verts_a = st.vertsA, *verts_b = st.vertsB;
    Plane *planes_a = st.planesA, *planes_b = st.planesB;
    {
        const Mat3x3 rot_a = Mat3x3::fromQuat(ps.aRot), rot_b = Mat3x3::fromQuat(ps.bRot);
        const Mat3x3 vm_a = rot_a * ps.aScale, vm_b = rot_b * ps.bScale;
        const Mat3x3 nm_a = rot_a * ps.aScale.inv(), nm_b = rot_b * ps.bScale.inv();
        const Vector3 a_pos = ps.aPos, b_pos = ps.bPos;
#pragma unroll 1
        for (u32 i = (u32)sub; i < nva + nvb; i += G) {
            if (i < nva) verts_a[i] = vm_a * am.vertices[i] + a_pos;
            else verts_b[i - nva] = vm_b * bm.vertices[i - nva] + b_pos;
        }
#pragma unroll 1
        for (u32 i = (u32)sub; i < nfa + nfb; i += G) {
            const bool is_a = i < nfa;
            const Plane local = is_a ? am.facePlanes[i] : bm.facePlanes[i - nfa];
            const Mat3x3 vm = is_a ? vm_a : vm_b;    // by value: a reference would put both in local memory
            const Mat3x3 nm = is_a ? nm_a : nm_b;
            const Vector3 on_plane = vm * (local.normal * local.d) + (is_a ? a_pos : b_pos);
            const Vector3 n = (nm * local.normal).normalize();
            (is_a ? planes_a[i] : planes_b[i - nfa]) = Plane { n, dot(n, on_plane) };
        }
    }
    __syncwarp(gm);
    // centre of A: vertex sum in index order (float addition is not associative)
    Vector3 center_a = Vector3::zero();
#pragma unroll 1
    for (u32 i = 0; i < nva; i++) center_a += verts_a[i];
    center_a /= (float)nva;

    // -- face queries (A's faces vs B, then B's vs A)
    const Winner fa = groupFaceQuery<G>(gm, sub, planes_a, nfa, verts_b, nvb);
    if (fa.sep > 0.0f) return false;
    const Winner fb = groupFaceQuery<G>(gm, sub, planes_b, nfb, verts_a, nva);
    if (fb.sep > 0.0f) return false;
    const float sep_a = fa.sep, sep_b = fb.sep;
    const i32 face_a = fa.idx, face_b = fb.idx;

    // -- edge query: edge pairs a-major over numHalfEdges/2 edges (half-edge 2k, twin
    // 2k+1), only pairs forming a face of the Minkowski difference are measured
    // (narrowphase.cpp:367-567); pair p = ia * eb + ib, lanes take p = sub, sub + G, ...
    const u32 ea = am.numHalfEdges / 2, eb = bm.numHalfEdges / 2;
    float e_sep = -FLT_MAX;
    i32 e_pair = 0x7fffffff;
    Vector3 e_normal = Vector3::zero();
#pragma unroll 1
    for (u32 p = (u32)sub; p < ea * eb; p += G) {
        const u32 ha = (p / eb) * 2, hb = (p % eb) * 2;
        const HalfEdge a0 = am.halfEdges[ha];
        const HalfEdge a1 = am.halfEdges[ha ^ 1u];
        const HalfEdge b0 = bm.halfEdges[hb];
        const HalfEdge b1 = bm.halfEdges[hb ^ 1u];
        float sep = -FLT_MAX;
        Vector3 normal = Vector3::zero();
        if (gaussMapArcsCross(planes_a[a0.face].normal, planes_a[a1.face].normal,
                              -planes_b[b0.face].normal, -planes_b[b1.face].normal)) {
            const Vector3 pa = verts_a[a0.rootVertex];
            const Vector3 qa = verts_a[am.halfEdges[a0.next].rootVertex];
            const Vector3 pb = verts_b[b0.rootVertex];
            const Vector3 qb = verts_b[bm.halfEdges[b0.next].rootVertex];
            const Vector3 axis = (qa - pa).cross(qb - pb);
            const float len2 = axis.length2();
            if (len2 != 0) {
                normal = axis * (1.f / sqrtf(len2));
                if (normal.dot(pa - center_a) < 0.0f) normal = -normal;
                sep = normal.dot(pb - pa);
            }
        }
        if (sep > e_sep) {
            e_sep = sep;
            e_pair = (i32)p;
            e_normal = normal;
            if (sep > 0) break;
        }
    }
    {
        const float my_sep = e_sep;
        const i32 my_pair = e_pair;
        const Winner ew = groupSequentialWinner<G>(gm, e_sep, e_pair, my_pair != 0x7fffffff);
        e_sep = ew.sep;
        e_pair = ew.idx;
        const unsigned owner = __ballot_sync(gm, my_pair == e_pair && my_pair != 0x7fffffff &&
                                                 my_sep == e_sep);
        if (owner) {
            const int src = __ffs(owner) - 1;
            e_normal.x = __shfl_sync(gm, e_normal.x, src);
            e_normal.y = __shfl_sync(gm, e_normal.y, src);
            e_normal.z = __shfl_sync(gm, e_normal.z, src);
        } else {
            // nothing beat the initial -FLT_MAX: the scalar scan keeps its defaults
            e_sep = -FLT_MAX;
            e_pair = 0;
            e_normal = Vector3::zero();
        }
    }
    if (e_sep > 0.0f) return false;

    // -- contact generation
    const bool face_contact_a = sep_a > e_sep;
    const bool face_contact_b = sep_b > e_sep;
    if (!face_contact_a && !face_contact_b) {
        // edge - edge: contact point on A's edge, depth = -separation, A is ref
        if (sub == 0) {
            const u32 ha = ((u32)e_pair / eb) * 2, hb = ((u32)e_pair % eb) * 2;
            const HalfEdge he_a = am.halfEdges[ha];
            const HalfEdge he_b = bm.halfEdges[hb];
            const Vector3 p = closestOnFirstSegment(
                verts_a[he_a.rootVertex], verts_a[am.halfEdges[he_a.next].rootVertex],
                verts_b[he_b.rootVertex], verts_b[bm.halfEdges[he_b.next].rootVertex]);
            writeSinglePointContact(out, ps.aArch, ps.aRow, ps.aInfo, ps.bArch, ps.bRow, ps.bInfo,
                                    p, e_normal, -e_sep);
        }
        return true;
    }
    const bool a_is_ref = sep_a >= sep_b;
    const Plane ref_plane = a_is_ref ? planes_a[face_a] : planes_b[face_b];
    const i32 ref_face = a_is_ref ? face_a : face_b;
    const HalfEdgeMesh &ref_mesh = a_is_ref ? am : bm;
    const HalfEdgeMesh &inc_mesh = a_is_ref ? bm : am;
    const Vector3 *ref_verts = a_is_ref ? verts_a : verts_b;
    const Vector3 *inc_verts = a_is_ref ? verts_b : verts_a;
    const i32 inc_face = groupMostOpposedFace<G>(gm, sub, a_is_ref ? planes_b : planes_a, a_is_ref ? nfb : nfa,
                                                 ref_plane.normal);
    if (inc_face == 0x7fffffff) return false;

    // incident polygon clipped against the side planes of the reference face
    // (normal = edge x n_ref), on the group's first lane; result in clipA (0) or clipB (1).
    // Either face over st.maxFaceVerts vertices, or a clipped polygon over st.clipCap points
    // (k-gon against k-gon: up to 2k), is an overflow: n = -1, and no contact.
    int n = 0, in_b = 0;
    if (sub == 0) {
        Vector3 *src = st.clipA, *dst = st.clipB;
        u32 he = inc_mesh.faceBaseHalfEdges[inc_face];
        u32 start = he;
        do {
            const HalfEdge cur = inc_mesh.halfEdges[he];
            he = cur.next;
            if (n == st.maxFaceVerts) {
                n = -1;
                break;
            }
            src[n++] = inc_verts[cur.rootVertex];
        } while (he != start);
        he = ref_mesh.faceBaseHalfEdges[ref_face];
        start = he;
        Vector3 cur_pt = ref_verts[ref_mesh.halfEdges[he].rootVertex];
        int sides = 0;
        while (n >= 0) {
            if (++sides > st.maxFaceVerts) {
                n = -1;
                break;
            }
            he = ref_mesh.halfEdges[he].next;
            Vector3 next_pt = ref_verts[ref_mesh.halfEdges[he].rootVertex];
            Vector3 side_n = cross(next_pt - cur_pt, ref_plane.normal);
            Plane side { side_n, dot(side_n, cur_pt) };
            cur_pt = next_pt;
            if (n > 0) n = clipAgainst(dst, side, src, n, st.clipCap);
            Vector3 *tmp = src;
            src = dst;
            dst = tmp;
            in_b ^= 1;
            if (he == start) break;
        }
        if (n < 0) atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
    }
    const int leader = __ffs(gm) - 1;
    n = __shfl_sync(gm, n, leader);
    if (n < 0) return false;
    in_b = __shfl_sync(gm, in_b, leader);
    __syncwarp(gm);
    const int count = groupManifold<G>(gm, sub, ref_plane, in_b ? st.clipB : st.clipA, n,
                                       in_b ? st.clipA : st.clipB, st.depths, out);
    if (count == 0) return false;
    if (sub == 0) {
        if (a_is_ref) writeContactHeader(out, ps.aArch, ps.aRow, ps.aInfo, ps.bArch, ps.bRow, ps.bInfo, count, ref_plane.normal);
        else writeContactHeader(out, ps.bArch, ps.bRow, ps.bInfo, ps.aArch, ps.aRow, ps.aInfo, count, ref_plane.normal);
    }
    return true;
}

// ---- narrowphase, dense over the candidates of ALL worlds ------------------------------------
// The contact of candidate i of world w lives in slot (w, i), so nothing here
// needs per-world ordering.  One launch per substep, a persistent grid of
// numSMs x (resident blocks per SM) blocks over the step's two work lists (built
// by the candidate search).  The unit of work is a warp item: kGroupLanes-lane
// groups on 4 hull - hull pairs, or kPlaneLanes-lane groups on 8 other pairs.
// Items are numbered [hull - hull items][other items], so the long chains start
// first, and handed out in that order by hullPairs' ticket (forEachTicket): both
// classes share every SM, neither waits for a wave of the other, and a warp that
// drew short pairs takes more.
// Each pair writes only its own contact slot and candHit entry, so which warp
// takes which pair changes no result.  orderContacts (prologue of the position
// solve) lists each world's hits in candidate order and assigns the dependency
// levels.
// Threads per block, measured on an H100 80GB HBM3 at a 700 W power limit (bench.py
// --steps 200 --warmup 20, means of 3 alternating runs, room / arena / room_render):
// 128 threads 1.3276 / 1.5689 / 10.983 ms/step, of which phys_narrowphase 0.347 /
// 0.295 / 0.622 ms; 64 threads 1.3284 / 1.5714 / 10.979 ms/step, phys_narrowphase
// 0.349 / 0.296 / 0.627 ms.
constexpr int kNarrowThreads = 128;
constexpr int kNarrowWarps = kNarrowThreads / 32;
// 640 / 512 resident threads per SM: the most that compile without local memory
// (96 / 128 registers)
constexpr int kNarrowMinBlocks = 640 / kNarrowThreads;
constexpr int kNarrowMinBlocksSpheres = 512 / kNarrowThreads;
// Lanes per hull - plane pair.  Measured on an H100 80GB HBM3 at a 400 W power limit
// (bench.py --steps 200, ms/step, room / arena / room_render): 4 lanes 1.376 / 1.596 /
// 11.66, 8 lanes 1.479 / 1.713 / 11.85.  With 2 lanes or 1 the room step took
// 2.0 / 1.9 ms.
constexpr int kPlaneLanes = 4;
constexpr int kHullPairsPerWarp = 32 / kGroupLanes;
constexpr int kPlanePairsPerWarp = 32 / kPlaneLanes;

// Hands the work items [0, items) out to the warps of a persistent grid (`warps` per
// block) by the ticket in `c`: one atomic per warp and item, fetched while the previous
// item runs.  The warp runs run(item) on all its lanes and syncs before its next item,
// which may reuse its staging.  Every warp has taken its last ticket before it counts
// itself out, so the last one out can zero the ticket and the finished count for the next
// launch.
template <typename Run>
__device__ __forceinline__ void forEachTicket(PairListCounters *c, const i32 items, const int warps,
                                              const int lane, Run &&run)
{
    i32 item = 0;
    if (lane == 0) item = atomicAdd(&c->ticket, 1);
    item = __shfl_sync(0xffffffffu, item, 0);
    while (item < items) {
        i32 next = 0;
        if (lane == 0) next = atomicAdd(&c->ticket, 1);    // in flight while this item runs
        run(item);
        __syncwarp();
        item = __shfl_sync(0xffffffffu, next, 0);
    }
    if (lane == 0 && atomicAdd(&c->finished, 1) == (i32)gridDim.x * warps - 1) {
        c->ticket = 0;
        c->finished = 0;
    }
}

template <bool SPHERE_HULL>
__global__ void __launch_bounds__(kNarrowThreads, SPHERE_HULL ? kNarrowMinBlocksSpheres : kNarrowMinBlocks)
physNarrowphaseKernel(EngineState *Sp)
{
    EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    fillColCache(S, P);
    // per warp: the scratch of its 4 hull - hull groups or of its 8 other groups
    __shared__ union {
        HullScratch hull[kHullPairsPerWarp];
        PlaneScratch plane[kPlanePairsPerWarp];
    } scratch[kNarrowWarps];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x / 32;
    const i32 num_hull = P.hullPairs.counters->count, num_other = P.otherPairs.counters->count;
    const i32 hull_items = (num_hull + kHullPairsPerWarp - 1) / kHullPairsPerWarp;
    const i32 items = hull_items + (num_other + kPlanePairsPerWarp - 1) / kPlanePairsPerWarp;
    // Both kinds of item share one copy of the pair's setup: with a copy per kind the
    // kernel needs more registers than its launch bounds allow and spills.
    forEachTicket(P.hullPairs.counters, items, kNarrowWarps, lane, [&](const i32 item) {
        const bool hull = item < hull_items;
        const int sub = hull ? lane % kGroupLanes : lane % kPlaneLanes;
        const int group = hull ? lane / kGroupLanes : lane / kPlaneLanes;
        const unsigned gm = hull ? ((1u << kGroupLanes) - 1u) << (group * kGroupLanes)
                                 : ((1u << kPlaneLanes) - 1u) << (group * kPlaneLanes);
        const i32 e = hull ? item * kHullPairsPerWarp + group : (item - hull_items) * kPlanePairsPerWarp + group;
        if (e >= (hull ? num_hull : num_other)) return;
        const PairEntry ent = (hull ? P.hullPairs : P.otherPairs).entries[e];
        const size_t slot = (size_t)ent.world * P.maxCandidatesPerWorld + ent.cand;
        const PairSetup ps = setupPair(worldObjects(S, P, ent.world), P.candidates[slot]);
        bool made = false;
        if (ps.test != 0) {
            if (hull) {
                made = hullHullGroup<kGroupLanes>(S, ps, smallHullStage(scratch[warp].hull[group]), gm, sub,
                                                  P.contacts[slot]);
            } else if (ps.test == PairHullPlane) {
                made = hullPlaneGroup<kPlaneLanes>(S, ps, scratch[warp].plane[group], gm, sub, P.contacts[slot]);
            } else {
                i32 hit = 0;
                if (sub == 0) hit = singlePointPair<SPHERE_HULL>(S, ps, P.contacts[slot]) ? 1 : 0;
                made = __shfl_sync(gm, hit, __ffs(gm) - 1) != 0;
            }
        }
        if (sub == 0) P.candHit[slot] = made ? 1 : 0;
    });
}

// ---- hulls past the staging caps: one warp per pair --------------------------------------
// With MADRONA_B200_MAX_HULL_SIZE = N > 16 and a primitive that needs it, the candidate
// search sends every pair with such a hull to PhysicsState::largePairs and each substep
// runs this kernel after the one above: the same group functions with all 32 lanes on one
// pair (the winner rules do not depend on the lane count, so the results are the scalar
// scan's), staging in dynamic shared memory sized from N instead of the fixed scratch --
// per warp both hulls' planes and vertices (2N x 16 B, 2N x 12 B), two clip buffers of 2N
// points and 2N depths: 112 N bytes, 3.5 KB at N = 32 and 27.9 KB at N = 255, where the 8
// warps of a block fill an SM's shared memory.  (A convex polygon of n points clipped by m
// side planes has at most n + m <= 2N; vertices that round onto a side plane can add a few,
// tests/test_large_hull_model.py, so clipAgainst keeps its "would not fit" return.)  The grid is what is resident at that size; pairs are handed out
// by a ticket as above, and each writes only its own contact slot and candHit entry.
constexpr int kLargeWarps = 8;
constexpr int kLargeThreads = 32 * kLargeWarps;
constexpr int kLargeStageBytesPerEntry = 2 * (int)(sizeof(Plane) + 3 * sizeof(Vector3) + sizeof(float));
static_assert(kLargeStageBytesPerEntry == 112, "large-hull stage layout");

__device__ __forceinline__ HullStage largeHullStage(unsigned char *base, const int n)
{
    Plane *planes = (Plane *)base;
    Vector3 *verts = (Vector3 *)(planes + 2 * n);
    Vector3 *clip_a = verts + 2 * n, *clip_b = clip_a + 2 * n;
    return HullStage { verts, verts + n, planes, planes + n, clip_a, clip_b, (float *)(clip_b + 2 * n),
                       n, n, n, 2 * n };
}

__global__ void __launch_bounds__(kLargeThreads, 1)
physNarrowphaseLargeKernel(EngineState *Sp)
{
    EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    fillColCache(S, P);
    extern __shared__ __align__(16) unsigned char large_stage[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x / 32;
    const int cap = P.maxHullSize;
    const HullStage st = largeHullStage(large_stage + (size_t)warp * cap * kLargeStageBytesPerEntry, cap);
    forEachTicket(P.largePairs.counters, P.largePairs.counters->count, kLargeWarps, lane, [&](const i32 item) {
        const PairEntry ent = P.largePairs.entries[item];
        const size_t slot = (size_t)ent.world * P.maxCandidatesPerWorld + ent.cand;
        const PairSetup ps = setupPair(worldObjects(S, P, ent.world), P.candidates[slot]);
        bool made = false;
        if (ps.test != 0) {
            // side a is a hull except in sphere - hull pairs, side b except in hull - plane pairs
            const HalfEdgeMesh *ha = ps.test != PairSphereHull ? &ps.aPrim->hull : nullptr;
            const HalfEdgeMesh *hb = ps.test != PairHullPlane ? &ps.bPrim->hull : nullptr;
            const bool fits = (!ha || (ha->numVertices <= (u32)cap && ha->numFaces <= (u32)cap)) &&
                              (!hb || (hb->numVertices <= (u32)cap && hb->numFaces <= (u32)cap));
            if (!fits || (ps.test != PairHullHull && ps.test != PairSphereHull && ps.test != PairHullPlane)) {
                if (lane == 0) atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
            } else if (ps.test == PairHullHull) {
                made = hullHullGroup<32>(S, ps, st, 0xffffffffu, lane, P.contacts[slot]);
            } else if (ps.test == PairHullPlane) {
                LargePlaneStage plane_stage { st.clipA, st.clipB, st.depths, st.maxFaceVerts };
                made = hullPlaneGroup<32>(S, ps, plane_stage, 0xffffffffu, lane, P.contacts[slot]);
            } else {
                const SphereHullResult r = sphereHullGroup<32>(ps.aPos, ps.aScale.d0 * ps.aPrim->sphereRadius, ps.bPos,
                                                               ps.bRot, ps.bScale, ps.bPrim->hull, st.vertsA,
                                                               0xffffffffu, lane);
                made = r.hit > 0;
                if (made && lane == 0) {
                    writeSinglePointContact(P.contacts[slot], ps.bArch, ps.bRow, ps.bInfo, ps.aArch, ps.aRow,
                                            ps.aInfo, r.point, r.normal, r.depth);
                }
            }
        }
        if (lane == 0) P.candHit[slot] = made ? 1 : 0;
    });
}

// ---- primitive classes, once before the launch graph is captured --------------------------
// The half-edge mesh does not store its largest face, so a primitive's class (PrimClass)
// comes from a walk over its faces.  The ObjectManager carries no primitive count either:
// physPrimExtentKernel takes it from the objects the bodies use, and checks that every
// world points at the ObjectManager of world 0, whose primitives the table describes.
// info[0] = primitives, info[1] = worlds with another ObjectManager, info[2] = primitives
// that are not small.
__global__ void __launch_bounds__(256)
physPrimExtentKernel(EngineState *Sp, i32 *info)
{
    const EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    const ObjectManager *first = &worldObjects(S, P, 0);
    const i32 tid = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
    for (i32 w = tid; w < (i32)S.numWorlds; w += stride) {
        if (&worldObjects(S, P, w) != first) atomicAdd(&info[1], 1);
    }
    for (u32 bi = 0; bi < P.numBodyArchetypes; bi++) {
        const BodyArchetype &b = P.bodies[bi];
        const TableDesc &t = S.tables[b.archetype];
        for (i32 row = tid; row < t.numRows; row += stride) {
            if (((const i32 *)t.columns[1])[row] < 0) continue;
            const i32 obj = bodyCol<i32>(S, b, PCObjectID, row);
            atomicMax(&info[0], (i32)(first->primOffsets[obj] + first->primCounts[obj]));
        }
    }
}

__global__ void __launch_bounds__(256)
physClassifyPrimsKernel(EngineState *Sp, unsigned char *classes, i32 num_prims, i32 *info)
{
    const EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    const i32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_prims) return;
    const CollisionPrimitive &prim = worldObjects(S, P, 0).prims[i];
    u32 cls = PrimSmall;
    if (prim.type == 2u) {
        const HalfEdgeMesh &m = prim.hull;
        // the longest face loop; a walk is bounded by the mesh's half-edges, so a broken
        // `next` chain cannot loop for ever (it then counts as a face of that length)
        u32 longest = 0;
        for (u32 f = 0; f < m.numFaces; f++) {
            const u32 start = m.faceBaseHalfEdges[f];
            u32 he = start, n = 0;
            do {
                he = m.halfEdges[he].next;
                n++;
            } while (he != start && he < m.numHalfEdges && n < m.numHalfEdges);
            if (n > longest) longest = n;
        }
        const u32 cap = (u32)P.maxHullSize;
        if (m.numVertices > cap || m.numFaces > cap || longest > cap) cls = PrimTooLarge;
        else if (m.numVertices > (u32)kMaxHullVerts || m.numFaces > (u32)kMaxHullFaces ||
                 longest > (u32)kMaxFaceVerts) cls = PrimLarge;
    }
    classes[i] = (unsigned char)cls;
    if (cls != PrimSmall) atomicAdd(&info[2], 1);
}

// Prologue of the position solve, run by the LPW lanes that own world w: list
// the world's contact slots in candidate order and give every contact its
// dependency level (see Contact::level) -- a sequential scan by the group's
// first lane over flags / body infos its lanes fetched in parallel.  The last level of
// each body slot is kept in `last_level` (shared, kMaxLevelBodies slots), or, for a world
// with more body slots when PhysicsState::levelScratch exists, in the world's row of it
// (up to maxWorldBodies slots).  A contact on a slot past the table is ordered after
// everything before it.
template <int LPW>
__device__ __forceinline__ void orderContacts(EngineState &S, const PhysicsState &P, const i32 w, const bool valid,
                                              const int lane, i32 *last_level /* [kMaxLevelBodies] of this world */)
{
    constexpr unsigned kGroupMask = LPW == 32 ? 0xffffffffu : ((1u << (LPW & 31)) - 1u);
    const int sub = lane & (LPW - 1);
    const int group_shift = (lane / LPW) * LPW;
    const unsigned gm = kGroupMask << group_shift;

    i32 num_slots = kMaxLevelBodies;
    if (P.levelScratch && valid) {
        i32 bodies = 0;
        for (u32 bi = 0; bi < P.numBodyArchetypes; bi++) bodies += S.tables[P.bodies[bi].archetype].worldCounts[w];
        if (bodies > kMaxLevelBodies) {
            last_level = P.levelScratch + (size_t)w * P.maxWorldBodies;
            num_slots = min(bodies, P.maxWorldBodies);
        }
    }
    for (int i = sub; i < num_slots; i += LPW) last_level[i] = 0;
    __syncwarp(gm);

    const i32 n = valid ? P.candCounts[w] : 0;
    const size_t base_slot = (size_t)w * P.maxCandidatesPerWorld;
    Contact *contacts = P.contacts + base_slot;
    i32 *order = P.contactOrder + (size_t)w * P.maxContactsPerWorld;
    i32 running = 0, max_level = 0, seq_level = 0;

    for (i32 base = 0; base < n; base += LPW) {
        const i32 i = base + sub;
        const bool hit = i < n && P.candHit[base_slot + i] != 0;
        u32 a = 0, b = 0;
        if (hit) {
            a = contacts[i].refInfo;
            b = contacts[i].altInfo;
        }
        const unsigned hits = (__ballot_sync(gm, hit) >> group_shift) & kGroupMask;
        i32 my_level = 0;
        unsigned todo = hits;
        while (todo) {
            const int src = __ffs(todo) - 1;
            todo &= todo - 1;
            const u32 sa_info = __shfl_sync(gm, a, group_shift + src);
            const u32 sb_info = __shfl_sync(gm, b, group_shift + src);
            i32 lvl = 0;
            if (sub == 0) {
                const u32 sa = sa_info >> 1, sb = sb_info >> 1;
                if (sa >= (u32)num_slots || sb >= (u32)num_slots) {
                    lvl = max_level + 1;          // unknown body: strictly after everything so far
                    seq_level = lvl;
                } else {
                    i32 dep = seq_level;
                    if (sa_info & 1u) dep = max(dep, last_level[sa]);
                    if (sb_info & 1u) dep = max(dep, last_level[sb]);
                    lvl = dep + 1;
                    if (sa_info & 1u) last_level[sa] = lvl;
                    if (sb_info & 1u) last_level[sb] = lvl;
                }
                if (lvl > max_level) max_level = lvl;
            }
            lvl = __shfl_sync(gm, lvl, group_shift);
            if (sub == src) my_level = lvl;
        }
        if (hit) {
            const i32 at = running + __popc(hits & ((1u << sub) - 1u));
            contacts[i].level = my_level;
            if (at < P.maxContactsPerWorld) order[at] = i;
        }
        running += __popc(hits);
    }
    if (valid && sub == 0) {
        if (running > P.maxContactsPerWorld) {
            atomicOr(&S.errorFlags, (u32)ErrPhysicsOverflow);
            running = P.maxContactsPerWorld;
        }
        P.contactCounts[w] = running;
        P.contactMaxLevel[w] = max_level;
    }
    __syncwarp(gm);
}

// =============================================================================================
// XPBD constraint solve (per world, sequential Gauss-Seidel in contact order)
// =============================================================================================

struct BodyPair {
    float invM1, invM2;
    Vector3 invI1, invI2;
};

__device__ __forceinline__ float positionalLambda(Vector3 tq1, Vector3 tq2, Vector3 ra1, Vector3 ra2,
                                                  float inv_m1, float inv_m2, float c, float alpha)
{
    float w1 = inv_m1 + dot(tq1, ra1);
    float w2 = inv_m2 + dot(tq2, ra2);
    return -c / (w1 + w2 + alpha);
}

__device__ __forceinline__ void applyPositional(Vector3 &x1, Vector3 &x2, Quat &q1, Quat &q2,
                                                Vector3 rot_axis1, Vector3 rot_axis2,
                                                float inv_m1, float inv_m2, Vector3 n, float lambda)
{
    x1 += lambda * inv_m1 * n;
    x2 -= lambda * inv_m2 * n;
    const float half = 0.5f * lambda;
    const Vector3 w1 = q1.rotateVec(half * rot_axis1);
    const Vector3 w2 = q2.rotateVec(half * rot_axis2);
    q1 += Quat::fromAngularVec(w1) * q1;
    q2 -= Quat::fromAngularVec(w2) * q2;
    q1 = q1.normalize();
    q2 = q2.normalize();
}

__device__ __forceinline__ float positionalCorrection(Vector3 &x1, Vector3 &x2, Quat &q1, Quat &q2,
                                                      Vector3 r1, Vector3 r2, const BodyPair &bp,
                                                      Vector3 n_world, float c, float alpha)
{
    const Vector3 n1 = q1.inv().rotateVec(n_world);
    const Vector3 n2 = q2.inv().rotateVec(n_world);
    const Vector3 tq1 = cross(r1, n1);
    const Vector3 tq2 = cross(r2, n2);
    const Vector3 ra1 = mulDiag(bp.invI1, tq1);
    const Vector3 ra2 = mulDiag(bp.invI2, tq2);
    const float lambda = positionalLambda(tq1, tq2, ra1, ra2, bp.invM1, bp.invM2, c, alpha);
    applyPositional(x1, x2, q1, q2, ra1, ra2, bp.invM1, bp.invM2, n_world, lambda);
    return lambda;
}

// depth-weighted mean contact point + deepest penetration (xpbd.cpp:421-449);
// false when all depths are zero
__device__ bool meanContact(const Contact &c, Vector3 *mean, float *deepest)
{
    float max_pen = -FLT_MAX, sum = 0.f;
    for (int i = 0; i < c.numPoints; i++) {
        float pen = c.points[i][3];
        if (pen > max_pen) max_pen = pen;
        sum += pen;
    }
    if (sum == 0.f) return false;
    Vector3 acc = Vector3::zero();
    for (int i = 0; i < c.numPoints; i++) {
        acc += c.points[i][3] / sum * Vector3 { c.points[i][0], c.points[i][1], c.points[i][2] };
    }
    *mean = acc;
    *deepest = max_pen;
    return true;
}

__device__ __forceinline__ void localArms(const PPosRot &pre1, const PPosRot &pre2, Vector3 p1, float depth,
                                          Vector3 n, Vector3 *r1, Vector3 *r2)
{
    const Vector3 p2 = p1 - n * depth;
    *r1 = pre1.q.inv().rotateVec(p1 - pre1.x);
    *r2 = pre2.q.inv().rotateVec(p2 - pre2.x);
}

// What the solves need of a body's object metadata, with its response type
// applied: a static body has no inverse mass or inertia.
struct BodyMass {
    float invM;
    Vector3 invI;
    float muS, muD;
};

__device__ __forceinline__ BodyMass loadBodyMass(const EngineState &S, const PhysicsState &P,
                                                 const ObjectManager &objs, u32 arch, i32 row)
{
    const RigidBodyMetadata m = objs.metadata[cachedCol<i32>(arch, PCObjectID, row)];
    BodyMass bm { m.invMass, m.invInertia, m.muS, m.muD };
    if (cachedCol<u32>(arch, PCResponseType, row) == kRespStatic) {
        bm.invM = 0.f;
        bm.invI = Vector3::zero();
    }
    return bm;
}

__device__ __forceinline__ BodyPair bodyPair(const BodyMass &m1, const BodyMass &m2, float *mu_s, float *mu_d)
{
    *mu_s = 0.5f * (m1.muS + m2.muS);
    *mu_d = 0.5f * (m1.muD + m2.muD);
    return BodyPair { m1.invM, m2.invM, m1.invI, m2.invI };
}

// ---- per-world body staging of the position solve ---------------------------------------------
// The position sweep and the joints read and rewrite the same few dozen bodies
// level after level.  The lanes that own a world first copy each body's x, q and
// BodyMass into shared memory; contacts and joints work on those copies, and the
// epilogue writes x, q back.  A body is staged when its world slot (worldBodySlot,
// also carried by Contact::refInfo / altInfo) is below kStagedBodies; the others,
// including bodies of unknown slot, are read and written in the global columns
// through the same accessors.  Staged or not depends on the slot alone, so every
// body has exactly one live copy during the solve and results do not depend on
// kStagedBodies.  Slots count rows awaiting compaction too: room (33 bodies) fits,
// arena's highest slots spill.  A block of 64 threads stages 32 * kPhysWarps /
// kPosSolverLanes worlds: 13.6 KB of static shared memory at 16 lanes per world.
constexpr int kStagedBodies = 48;

struct PosBody {                // x, q read / write
    Vector3 x;
    Quat q;
    BodyMass m;
};

__device__ __forceinline__ bool isStaged(u32 info) { return (info >> 1) < (u32)kStagedBodies; }

__device__ __forceinline__ PosBody globalPosBody(const EngineState &S, const PhysicsState &P,
                                                 const ObjectManager &objs, u32 arch, i32 row)
{
    return PosBody { cachedCol<Vector3>(arch, PCPosition, row), cachedCol<Quat>(arch, PCRotation, row),
                     loadBodyMass(S, P, objs, arch, row) };
}

// info: (slot << 1) | mutable, as in Contact::refInfo
__device__ __forceinline__ PosBody loadPosBody(const EngineState &S, const PhysicsState &P,
                                               const ObjectManager &objs, const PosBody *stage,
                                               u32 info, u32 arch, i32 row)
{
    return isStaged(info) ? stage[info >> 1] : globalPosBody(S, P, objs, arch, row);
}

__device__ __forceinline__ void storePosBody(const EngineState &S, const PhysicsState &P, PosBody *stage,
                                             u32 info, u32 arch, i32 row, Vector3 x, Quat q)
{
    if (isStaged(info)) {
        stage[info >> 1].x = x;
        stage[info >> 1].q = q;
    } else {
        cachedCol<Vector3>(arch, PCPosition, row) = x;
        cachedCol<Quat>(arch, PCRotation, row) = q;
    }
}

// fn(slot, arch, row) for every live body of world w with a staged slot, spread
// over the LPW lanes (sub = lane in group) that own w
template <int LPW, typename Fn>
__device__ __forceinline__ void forEachStagedBody(const EngineState &S, const PhysicsState &P, const i32 w,
                                                  const int sub, Fn &&fn)
{
    for (u32 bi = 0; bi < P.numBodyArchetypes; bi++) {
        const u32 arch = P.bodies[bi].archetype;
        const TableDesc &t = S.tables[arch];
        const i32 first = t.worldOffsets[w];
        const i32 end = first + t.worldCounts[w];
        const i32 *world_col = (const i32 *)t.columns[1];
        for (i32 row = first + sub; row < end; row += LPW) {
            if (world_col[row] != w) continue;   // destroyed, awaiting compaction
            const i32 slot = worldBodySlot(S, P, w, arch, row);
            if ((u32)slot < (u32)kStagedBodies) fn(slot, arch, row);
        }
    }
}

// normal push-out along the contact normal + static friction (xpbd.cpp:347-419, 454-550)
__device__ void solveContactPosition(EngineState &S, const PhysicsState &P, const ObjectManager &objs,
                                     PosBody *stage, Contact &c)
{
    c.lambdaN = 0.f;

    const PosBody b1 = loadPosBody(S, P, objs, stage, c.refInfo, c.refArch, c.refRow);
    const PosBody b2 = loadPosBody(S, P, objs, stage, c.altInfo, c.altArch, c.altRow);
    const PPosRot prev1 = cachedCol<PPosRot>(c.refArch, PCPrevState, c.refRow);
    const PPosRot prev2 = cachedCol<PPosRot>(c.altArch, PCPrevState, c.altRow);
    const PPosRot pre1 = cachedCol<PPosRot>(c.refArch, PCPreSolvePos, c.refRow);
    const PPosRot pre2 = cachedCol<PPosRot>(c.altArch, PCPreSolvePos, c.altRow);

    float mu_s, mu_d;
    const BodyPair bp = bodyPair(b1.m, b2.m, &mu_s, &mu_d);

    Vector3 x1 = b1.x, x2 = b2.x;
    Quat q1 = b1.q, q2 = b2.q;

    Vector3 mean;
    float deepest;
    if (!meanContact(c, &mean, &deepest)) return;

    const Vector3 n { c.normal.x, c.normal.y, c.normal.z };
    Vector3 r1, r2;
    localArms(pre1, pre2, mean, deepest, n, &r1, &r2);

    Vector3 p1 = q1.rotateVec(r1) + x1;
    Vector3 p2 = q2.rotateVec(r2) + x2;
    const float d = dot(p1 - p2, n);
    if (d > 0) {
        const float lambda_n = positionalCorrection(x1, x2, q1, q2, r1, r2, bp, n, d, 0);
        c.lambdaN = lambda_n;

        const Vector3 p1_hat = prev1.q.rotateVec(r1) + prev1.x;
        const Vector3 p2_hat = prev2.q.rotateVec(r2) + prev2.x;
        p1 = q1.rotateVec(r1) + x1;
        p2 = q2.rotateVec(r2) + x2;
        const Vector3 dp = (p1 - p1_hat) - (p2 - p2_hat);
        const Vector3 dp_t = dp - dot(dp, n) * n;
        const float slide = dp_t.length();
        if (slide > 0.f) {
            const Vector3 t_world = dp_t / slide;
            const Vector3 t1 = q1.inv().rotateVec(t_world);
            const Vector3 t2 = q2.inv().rotateVec(t_world);
            const Vector3 tq1 = cross(r1, t1);
            const Vector3 tq2 = cross(r2, t2);
            const Vector3 ra1 = mulDiag(bp.invI1, tq1);
            const Vector3 ra2 = mulDiag(bp.invI2, tq2);
            const float lambda_t = positionalLambda(tq1, tq2, ra1, ra2, bp.invM1, bp.invM2, slide, 0);
            if (lambda_t > lambda_n * mu_s) {
                applyPositional(x1, x2, q1, q2, ra1, ra2, bp.invM1, bp.invM2, t_world, lambda_t);
            }
        }
    }

    storePosBody(S, P, stage, c.refInfo, c.refArch, c.refRow, x1, q1);
    storePosBody(S, P, stage, c.altInfo, c.altArch, c.altRow, x2, q2);
}

__device__ void angularCorrection(Quat &q1, Quat &q2, const BodyPair &bp, Vector3 axis_world, float theta)
{
    const Vector3 n1 = q1.inv().rotateVec(axis_world);
    const Vector3 n2 = q2.inv().rotateVec(axis_world);
    const Vector3 ra1 = mulDiag(bp.invI1, n1);
    const Vector3 ra2 = mulDiag(bp.invI2, n2);
    const float w1 = dot(n1, ra1);
    const float w2 = dot(n2, ra2);
    const float lambda = -theta / (w1 + w2 + 0);
    const float half = 0.5f * lambda;
    const Quat u1 = Quat::fromAngularVec(q1.rotateVec(half * ra1));
    const Quat u2 = Quat::fromAngularVec(q2.rotateVec(half * ra2));
    q1 = (q1 + u1 * q1).normalize();
    q2 = (q2 - u2 * q2).normalize();
}

// fixed / hinge joints (xpbd.cpp:552-718)
__device__ void solveJoint(EngineState &S, const PhysicsState &P, const ObjectManager &objs,
                           PosBody *stage, const i32 w, const PJoint &j)
{
    if (j.e1ID < 0 || j.e2ID < 0 || j.e1ID >= S.entityCapacity || j.e2ID >= S.entityCapacity) return;
    const EntitySlot s1 = S.entitySlots[j.e1ID];
    const EntitySlot s2 = S.entitySlots[j.e2ID];
    if (s1.gen != j.e1Gen || s2.gen != j.e2Gen) return;
    const u32 a1 = (u32)s1.a, a2 = (u32)s2.a;
    const i32 r1row = s1.b, r2row = s2.b;
    if (!isBodyArchetype(a1) || !isBodyArchetype(a2)) return;
    // slot info as in Contact::refInfo (the mutable bit is not read here)
    const u32 info1 = (u32)worldBodySlot(S, P, w, a1, r1row) << 1;
    const u32 info2 = (u32)worldBodySlot(S, P, w, a2, r2row) << 1;

    const PosBody b1 = loadPosBody(S, P, objs, stage, info1, a1, r1row);
    const PosBody b2 = loadPosBody(S, P, objs, stage, info2, a2, r2row);
    Vector3 x1 = b1.x, x2 = b2.x;
    Quat q1 = b1.q, q2 = b2.q;

    float mu_s, mu_d;
    const BodyPair bp = bodyPair(b1.m, b2.m, &mu_s, &mu_d);

    Vector3 correction;
    if (j.type == 0) {
        const Quat o1 = (q1 * j.fixed.attachRot1).normalize();
        const Quat o2 = (q2 * j.fixed.attachRot2).normalize();
        const Quat diff = o1 * o2.inv();
        Vector3 dq = 2.f * Vector3 { diff.x, diff.y, diff.z };
        const float mag = dq.length();
        if (mag > 0) {
            dq /= mag;
            angularCorrection(q1, q2, bp, dq, mag);
        }
        const Vector3 p1 = q1.rotateVec(j.r1) + x1;
        const Vector3 p2 = q2.rotateVec(j.r2) + x2;
        const Vector3 delta = p2 - p1;
        const Quat frame = (q1 * j.fixed.attachRot1).normalize();
        const Vector3 ax_a = frame.rotateVec(madrona::math::fwd);
        const Vector3 ax_b = frame.rotateVec(madrona::math::right);
        const Vector3 ax_c = cross(ax_a, ax_b);
        correction = Vector3::zero();
        correction -= (dot(delta, ax_a) - j.fixed.separation) * ax_a;
        correction -= dot(delta, ax_b) * ax_b;
        correction -= dot(delta, ax_c) * ax_c;
    } else {
        const Vector3 w1 = q1.rotateVec(j.hinge.a1Local);
        const Vector3 w2 = q2.rotateVec(j.hinge.a2Local);
        Vector3 dq = cross(w1, w2);
        const float mag = dq.length();
        if (mag > 0) {
            dq /= mag;
            angularCorrection(q1, q2, bp, dq, mag);
        }
        const Vector3 p1 = q1.rotateVec(j.r1) + x1;
        const Vector3 p2 = q2.rotateVec(j.r2) + x2;
        correction = p2 - p1;
    }

    const float cmag = correction.length();
    if (cmag > 0.f) {
        correction /= cmag;
        positionalCorrection(x1, x2, q1, q2, j.r1, j.r2, bp, correction, cmag, 0);
    }
    storePosBody(S, P, stage, info1, a1, r1row, x1, q1);
    storePosBody(S, P, stage, info2, a2, r2row, x2, q2);
}

// Contact sweep of one world by a group of LPW lanes (32 / LPW worlds share a
// warp).  Contacts are swept level by level (Contact::level): the contacts of a
// level run concurrently, levels run in order -- same floats as the reference's
// one-thread-per-world sequential sweep (xpbd.cpp:720-736).  Contacts are taken
// in chunks of 32, chunk-major: a later chunk only holds later contacts and the
// levels inside a chunk run in order, so any two contacts sharing a mutable body
// keep their sequential order.  Inside a level the members are compacted onto
// the group's first lanes (ballot + find-nth-set).
// Several worlds per warp multiply the worlds in flight per SM at no register
// cost.  Measured on room at 8192 worlds (H100, staged position solve, both solves
// at 16 lanes): 16 lanes per world 1.515 ms/step (position solve 0.371, velocity
// solve 0.256 ms/step), both at 8 lanes 1.537 (0.426, 0.225).  So each solve has its
// own lane count.  The position solve keeps 16 lanes: a level's contacts spread over
// more lanes, and 4 lanes does not fit (16 staged worlds per block exceed 48 KB of
// static shared memory).  The velocity solve fits 8 blocks of 64 threads per SM
// (121 registers at 16 lanes, 128 at 8): 32 worlds per SM at 16 lanes, 64 at 8.
// velocitySolveLanes keeps 16 lanes while the worlds fit one wave of that (arena:
// 4096 worlds on 132 SMs) and takes 8 past it (room: 8192 worlds in one wave
// instead of two).
constexpr int kPosSolverLanes = 16;
constexpr int kVelSolveBlocksPerSM = 8;

template <int LPW, typename Fn>
__device__ __forceinline__ void sweepContactLevels(const Contact *contacts, const i32 *order, const i32 n,
                                                   const i32 levels, const int lane, Fn &&solve)
{
    constexpr int kPerLane = 32 / LPW;
    constexpr unsigned kGroupMask = LPW == 32 ? 0xffffffffu : ((1u << (LPW & 31)) - 1u);
    const int sub = lane & (LPW - 1);
    const int group_shift = (lane / LPW) * LPW;

    i32 n_max = n, levels_max = levels;
#pragma unroll
    for (int o = LPW; o < 32; o <<= 1) {
        n_max = max(n_max, __shfl_xor_sync(0xffffffffu, n_max, o));
        levels_max = max(levels_max, __shfl_xor_sync(0xffffffffu, levels_max, o));
    }

    for (i32 base = 0; base < n_max; base += 32) {
        i32 lv[kPerLane];
#pragma unroll
        for (int r = 0; r < kPerLane; r++) {
            const i32 i = base + r * LPW + sub;
            lv[r] = i < n ? contacts[order[i]].level : 0;
        }
        for (i32 lvl = 1; lvl <= levels_max; lvl++) {
            unsigned members = 0;
#pragma unroll
            for (int r = 0; r < kPerLane; r++) {
                const unsigned b = __ballot_sync(0xffffffffu, lv[r] == lvl);
                members |= ((b >> group_shift) & kGroupMask) << (r * LPW);
            }
            const int count = __popc(members);
            for (int k = sub; k < count; k += LPW) {
                // member bit m = r * LPW + lane-in-group: fetch that lane's slot[r]
                const int m = (int)__fns(members, 0, k + 1);
                solve(order[base + m]);
            }
            __syncwarp();
        }
    }
}

// Joints follow the contacts, sequentially.  stage: [kStagedBodies] of world w.
__device__ void phaseSolvePositions(EngineState &S, const PhysicsState &P, const i32 w, const bool valid,
                                    const int lane, PosBody *stage)
{
    const ObjectManager &objs = worldObjects(S, P, w);
    const int sub = lane & (kPosSolverLanes - 1);
    if (valid) {
        forEachStagedBody<kPosSolverLanes>(S, P, w, sub, [&](i32 slot, u32 arch, i32 row) {
            stage[slot] = globalPosBody(S, P, objs, arch, row);
        });
    }
    __syncwarp();

    Contact *contacts = P.contacts + (size_t)w * P.maxCandidatesPerWorld;
    const i32 *order = P.contactOrder + (size_t)w * P.maxContactsPerWorld;
    const i32 n = valid ? P.contactCounts[w] : 0;
    const i32 levels = valid ? P.contactMaxLevel[w] : 0;
    sweepContactLevels<kPosSolverLanes>(contacts, order, n, levels, lane, [&](i32 i) {
        solveContactPosition(S, P, objs, stage, contacts[i]);
    });

    const TableDesc &jt = S.tables[P.jointArchetype];
    if (valid && sub == 0 && jt.numRows > 0) {
        const PJoint *joints = (const PJoint *)jt.columns[P.jointCol];
        const i32 *jw = (const i32 *)jt.columns[1];
        const i32 first = jt.worldOffsets[w];
        const i32 count = jt.worldCounts[w];
        for (i32 r = first; r < first + count; r++) {
            if (jw[r] < 0) continue;
            solveJoint(S, P, objs, stage, w, joints[r]);
        }
    }
    __syncwarp();

    if (valid) {
        forEachStagedBody<kPosSolverLanes>(S, P, w, sub, [&](i32 slot, u32 arch, i32 row) {
            cachedCol<Vector3>(arch, PCPosition, row) = stage[slot].x;
            cachedCol<Quat>(arch, PCRotation, row) = stage[slot].q;
        });
    }
}

__device__ __forceinline__ Vector3 relativeVelocity(Vector3 v1, Vector3 v2, Vector3 o1, Vector3 o2,
                                                    Vector3 d1, Vector3 d2)
{
    return (v1 + cross(o1, d1)) - (v2 + cross(o2, d2));
}

// restitution on the mean contact, then dynamic friction per contact point
// (xpbd.cpp:781-1039)
__device__ void solveContactVelocity(EngineState &S, const PhysicsState &P, const ObjectManager &objs,
                                     const Contact &c, float h, float restitution_threshold)
{
    PVelocity &vel1_ref = cachedCol<PVelocity>(c.refArch, PCVelocity, c.refRow);
    PVelocity &vel2_ref = cachedCol<PVelocity>(c.altArch, PCVelocity, c.altRow);
    const Quat q1 = cachedCol<Quat>(c.refArch, PCRotation, c.refRow);
    const Quat q2 = cachedCol<Quat>(c.altArch, PCRotation, c.altRow);
    const PPosRot pre1 = cachedCol<PPosRot>(c.refArch, PCPreSolvePos, c.refRow);
    const PPosRot pre2 = cachedCol<PPosRot>(c.altArch, PCPreSolvePos, c.altRow);
    const PVelocity pv1 = cachedCol<PVelocity>(c.refArch, PCPreSolveVel, c.refRow);
    const PVelocity pv2 = cachedCol<PVelocity>(c.altArch, PCPreSolveVel, c.altRow);

    float mu_s, mu_d;
    const BodyPair bp = bodyPair(loadBodyMass(S, P, objs, c.refArch, c.refRow),
                                 loadBodyMass(S, P, objs, c.altArch, c.altRow), &mu_s, &mu_d);

    Vector3 v1 = vel1_ref.linear, o1 = vel1_ref.angular;
    Vector3 v2 = vel2_ref.linear, o2 = vel2_ref.angular;
    const Vector3 n { c.normal.x, c.normal.y, c.normal.z };

    {
        Vector3 mean;
        float deepest;
        if (!meanContact(c, &mean, &deepest)) return;
        Vector3 r1, r2;
        localArms(pre1, pre2, mean, deepest, n, &r1, &r2);

        const Vector3 v_bar = relativeVelocity(pv1.linear, pv2.linear, pv1.angular, pv2.angular,
                                               pre1.q.rotateVec(r1), pre2.q.rotateVec(r2));
        const float vn_bar = dot(n, v_bar);
        const Vector3 r1_world = q1.rotateVec(r1);
        const Vector3 r2_world = q2.rotateVec(r2);
        const Vector3 tq1 = cross(r1, q1.inv().rotateVec(n));
        const Vector3 tq2 = cross(r2, q2.inv().rotateVec(n));

        const Vector3 v = relativeVelocity(v1, v2, o1, o2, r1_world, r2_world);
        const float vn = dot(n, v);
        float e = 0.3f;
        if (fabsf(vn_bar) <= restitution_threshold) e = 0.f;
        const float target = fminf(-e * vn_bar, 0) - vn;
        const Vector3 ra1 = mulDiag(bp.invI1, tq1);
        const Vector3 ra2 = mulDiag(bp.invI2, tq2);
        const float w1 = bp.invM1 + dot(tq1, ra1);
        const float w2 = bp.invM2 + dot(tq2, ra2);
        const float inv_w = 1.f / (w1 + w2);
        const float impulse = target * inv_w;
        if (impulse != 0.f) {
            v1 += n * impulse * bp.invM1;
            v2 -= n * impulse * bp.invM2;
            o1 += q1.rotateVec(impulse * ra1);
            o2 -= q2.rotateVec(impulse * ra2);
        }
    }

    float pen_sum = 0.f;
    for (int i = 0; i < c.numPoints; i++) pen_sum += c.points[i][3];

    for (int i = 0; i < c.numPoints; i++) {
        Vector3 r1, r2;
        localArms(pre1, pre2, Vector3 { c.points[i][0], c.points[i][1], c.points[i][2] },
                  c.points[i][3], n, &r1, &r2);
        const Vector3 r1_world = q1.rotateVec(r1);
        const Vector3 r2_world = q2.rotateVec(r2);
        const float lambda = c.lambdaN * (c.points[i][3] / pen_sum);

        const Vector3 v = relativeVelocity(v1, v2, o1, o2, r1_world, r2_world);
        const float vn = dot(n, v);
        const Vector3 vt = v - n * vn;
        const float vt_len = vt.length();
        if (vt_len == 0.f) continue;
        const Vector3 dir = vt / vt_len;
        const Vector3 d1 = q1.inv().rotateVec(dir);
        const Vector3 d2 = q2.inv().rotateVec(dir);
        const Vector3 tq1 = cross(r1, d1);
        const Vector3 tq2 = cross(r2, d2);
        const Vector3 ra1 = mulDiag(bp.invI1, tq1);
        const Vector3 ra2 = mulDiag(bp.invI2, tq2);
        const float w1 = bp.invM1 + dot(tq1, ra1);
        const float w2 = bp.invM2 + dot(tq2, ra2);
        const float inv_w = 1.f / (w1 + w2);
        const float friction = mu_d * fabsf(lambda) * inv_w / h;
        const float corrected = -fminf(friction, vt_len);
        const float impulse = corrected * inv_w;
        if (impulse == 0.f) continue;
        v1 += dir * impulse * bp.invM1;
        v2 -= dir * impulse * bp.invM2;
        o1 += q1.rotateVec(impulse * ra1);
        o2 -= q2.rotateVec(impulse * ra2);
    }

    vel1_ref = PVelocity { v1, o1 };
    vel2_ref = PVelocity { v2, o2 };
}

// Not staged: with the velocity sweep's shorter load chains, copying every body
// in and out cost more than the sweep saved (DESIGN.md 3.2).
template <int LPW>
__device__ void phaseSolveVelocities(EngineState &S, const PhysicsState &P, const i32 w, const bool valid,
                                     const int lane)
{
    const ObjectManager &objs = worldObjects(S, P, w);
    const PhysicsWorldParams &params = worldParams(S, P, w);
    const Contact *contacts = P.contacts + (size_t)w * P.maxCandidatesPerWorld;
    const i32 *order = P.contactOrder + (size_t)w * P.maxContactsPerWorld;
    const i32 n = valid ? P.contactCounts[w] : 0;
    const i32 levels = valid ? P.contactMaxLevel[w] : 0;
    sweepContactLevels<LPW>(contacts, order, n, levels, lane, [&](i32 i) {
        solveContactVelocity(S, P, objs, contacts[i], params.h, params.restitutionThreshold);
    });
}

// =============================================================================================
// Launchers.  Row-parallel phases (leaf update + refit, integrate, velocity
// update) are grid-stride kernels over all rows of every body archetype; the
// candidate search gives each world a warp, the solves give each world
// kPosSolverLanes / velocitySolveLanes lanes (and the position solve a shared-memory
// copy of its bodies, kStagedBodies).
// (A single fused warp-per-world kernel for the whole step would spread its warps
// over every phase of a large instruction footprint, and the light phases would
// inherit the narrowphase's register count and occupancy.)
// =============================================================================================

// ops of physBodyKernel
enum PhysPhase : u32 {
    PhaseUpdateLeaves = 1, PhaseIntegrate, PhaseSetVelocities, PhaseTGSVelocities, PhaseTGSPositions,
};

// registers unconstrained (at most 1 block per SM is promised); bodyGrid launches 4 blocks per SM
template <u32 OP>
__global__ void __launch_bounds__(256, 1)
physBodyKernel(EngineState *Sp)
{
    const EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    if (blockIdx.y >= P.numBodyArchetypes) return;
    const BodyArchetype &b = P.bodies[blockIdx.y];
    const TableDesc &t = S.tables[b.archetype];
    const i32 n = t.numRows;
    const i32 *world_col = (const i32 *)t.columns[1];
    for (i32 row = blockIdx.x * blockDim.x + threadIdx.x; row < n; row += gridDim.x * blockDim.x) {
        const i32 w = world_col[row];
        if (w < 0) continue;
        if constexpr (OP == PhaseUpdateLeaves) {
            // leaf update, then straight into the refit of that leaf (it only
            // needs the leaf's own new box) -- unless the world asked for a
            // rebuild, whose thread refits all leaves afterwards
            rowUpdateLeaf(S, P, b, row, w);
            if (!worldBVH(S, P, w).forceRebuild) rowRefit(S, P, b, row, w);
        }
        else if constexpr (OP == PhaseIntegrate) rowIntegrate(S, P, b, row, w);
        else if constexpr (OP == PhaseSetVelocities) rowSetVelocity(S, P, b, row, w);
        else if constexpr (OP == PhaseTGSVelocities) rowTGSVelocities(S, P, b, row, w);
        else if constexpr (OP == PhaseTGSPositions) rowTGSPositions(S, P, b, row, w);
    }
}

__global__ void __launch_bounds__(128)
physRebuildKernel(EngineState *Sp)
{
    EngineState &S = *Sp;
    const i32 w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= (i32)S.numWorlds) return;
    phaseRebuild(S, *S.physics, w);
}

// The per-world kernels run kPhysWarps warps per block: one world per warp in the
// candidate search, 32 / kPosSolverLanes resp. 32 / velocitySolveLanes worlds per
// warp in the solves.
constexpr int kPhysWorldThreads = 32 * kPhysWarps;

__global__ void __launch_bounds__(kPhysWorldThreads, 8)
physFindCandidatesKernel(EngineState *Sp)
{
    EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    fillColCache(S, P);
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const i32 w = (i32)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (w >= (i32)S.numWorlds) return;
    __shared__ CandidateScratch cand_scratch;
    phaseFindCandidates(S, P, w, lane, warp, cand_scratch);
}

// forEachTicket for a whole block: thread 0 draws the tickets, every thread runs run(item)
// and the block syncs before the next item, which may reuse its shared memory.
template <typename Run>
__device__ __forceinline__ void forEachBlockTicket(PairListCounters *c, const i32 items, i32 *slot, Run &&run)
{
    if (threadIdx.x == 0) *slot = atomicAdd(&c->ticket, 1);
    __syncthreads();
    i32 item = *slot;
    while (item < items) {
        __syncthreads();     // every thread has read the slot
        if (threadIdx.x == 0) *slot = atomicAdd(&c->ticket, 1);    // in flight while this item runs
        run(item);
        __syncthreads();
        item = *slot;
    }
    if (threadIdx.x == 0 && atomicAdd(&c->finished, 1) == (i32)gridDim.x - 1) {
        c->ticket = 0;
        c->finished = 0;
    }
}

// Launched right after physFindCandidatesKernel when MADRONA_B200_MAX_BODIES_PER_WORLD > 128:
// a persistent grid over the worlds that kernel listed, one block per world.
__global__ void __launch_bounds__(kLargeSearchThreads, 1)
physFindCandidatesLargeKernel(EngineState *Sp)
{
    EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    fillColCache(S, P);
    __shared__ LargeSearchScratch scratch;
    forEachBlockTicket(P.largeWorlds.counters, P.largeWorlds.counters->count, &scratch.ticket, [&](const i32 item) {
        phaseFindCandidatesLarge(S, P, P.largeWorlds.entries[item].world, scratch);
    });
}

// LPW lanes per world.  The lanes of a warp past the last world idle along on the
// last world (valid = false); returns false when the whole warp is past it.
template <int LPW>
__device__ __forceinline__ bool solverWorld(const EngineState &S, i32 &w, bool &valid)
{
    const i32 first_w = (i32)((blockIdx.x * blockDim.x + (threadIdx.x & ~31u)) / LPW);
    if (first_w >= (i32)S.numWorlds) return false;
    const i32 my_w = (i32)((blockIdx.x * blockDim.x + threadIdx.x) / LPW);
    valid = my_w < (i32)S.numWorlds;
    w = valid ? my_w : (i32)S.numWorlds - 1;
    return true;
}

// physicsHostAfterRegistry sets this kernel's carveout to kPosSolveCarveoutPercent: 132 KB of
// the SM's 228 KB maximum, the smallest H100 configuration that holds its 8 blocks (static
// stage + the 1 KB the driver reserves per block).  The other 124 KB of the SM's 256 KB stay
// L1, which keeps the contacts and the PreSolvePositional / SubstepPrevState rows that every
// level of a world re-reads.  Measured on room at 8192 worlds (H100 80GB HBM3, 700 W): the
// node took 0.342 ms/step with the maximum carveout, 0.303 at 164 KB, 0.289 at 132 KB.
constexpr int kPosSolveCarveoutPercent = 58;
static_assert(8 * (sizeof(ColCache) + (kPhysWorldThreads / kPosSolverLanes) *
                   (sizeof(i32) * kMaxLevelBodies + sizeof(PosBody) * kStagedBodies) + 1024) <= 132 * 1024,
              "8 position-solve blocks no longer fit the 132 KB shared-memory configuration");

__global__ void __launch_bounds__(kPhysWorldThreads, 8)
physSolvePositionsKernel(EngineState *Sp)
{
    EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    fillColCache(S, P);
    const int lane = threadIdx.x & 31;
    i32 w;
    bool valid;
    if (!solverWorld<kPosSolverLanes>(S, w, valid)) return;
    constexpr int kWorldsPerBlock = kPhysWorldThreads / kPosSolverLanes;
    __shared__ i32 last_level[kWorldsPerBlock][kMaxLevelBodies];
    __shared__ PosBody pos_stage[kWorldsPerBlock][kStagedBodies];
    orderContacts<kPosSolverLanes>(S, P, w, valid, lane, last_level[threadIdx.x / kPosSolverLanes]);
    phaseSolvePositions(S, P, w, valid, lane, pos_stage[threadIdx.x / kPosSolverLanes]);
}

template <int LPW>
__global__ void __launch_bounds__(kPhysWorldThreads, kVelSolveBlocksPerSM)
physSolveVelocitiesKernel(EngineState *Sp)
{
    EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    fillColCache(S, P);
    const int lane = threadIdx.x & 31;
    i32 w;
    bool valid;
    if (!solverWorld<LPW>(S, w, valid)) return;
    phaseSolveVelocities<LPW>(S, P, w, valid, lane);
}

// =============================================================================================
// Standalone overlap rows (setupStandaloneBroadphaseOverlapTasks): the step's candidate list
// as the CandidateTemporary table the reference's findIntersectingEntry fills
// (broadphase.cpp:930-993), world-major, each world in candidate (== CPU) order.  The node
// replaces the table's rows; setupStandaloneBroadphaseCleanupTasks clears them again.
// =============================================================================================

constexpr int kEmitScanThreads = 1024;

// 1 block: exclusive scan of candCounts over all worlds -> worldOffsets / worldCounts /
// numRows.  Rows past the table's capacity are dropped (ErrTableOverflow); highWater keeps
// the full demand so the host grows the table before the next step.
__global__ void __launch_bounds__(kEmitScanThreads)
physEmitOverlapsScanKernel(EngineState *Sp, u32 archetype)
{
    EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    TableDesc &t = S.tables[archetype];
    const i32 W = (i32)S.numWorlds;
    const i32 per = (W + kEmitScanThreads - 1) / kEmitScanThreads;
    const i32 first = min(W, (i32)threadIdx.x * per), last = min(W, first + per);
    i32 sum = 0;
    for (i32 w = first; w < last; w++) sum += P.candCounts[w];

    __shared__ i32 warp_incl[kEmitScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    i32 incl = sum;
    for (int o = 1; o < 32; o <<= 1) {
        const i32 up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
    }
    if (lane == 31) warp_incl[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        i32 v = warp_incl[lane];
        for (int o = 1; o < 32; o <<= 1) {
            const i32 up = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += up;
        }
        warp_incl[lane] = v;
    }
    __syncthreads();
    i32 off = incl - sum + (warp > 0 ? warp_incl[warp - 1] : 0);
    const i32 total = warp_incl[kEmitScanThreads / 32 - 1];
    const i32 cap = t.capacity;
    for (i32 w = first; w < last; w++) {
        const i32 n = P.candCounts[w];
        const i32 o = min(off, cap);
        t.worldOffsets[w] = o;
        t.worldCounts[w] = min(off + n, cap) - o;
        off += n;
    }
    if (threadIdx.x == 0) {
        t.numRows = min(total, cap);
        t.needsSort = 0;
        if ((u32)total > t.highWater) t.highWater = (u32)total;
        if (total > cap) {
            atomicOr(&S.errorFlags, (u32)ErrTableOverflow);
            S.errorArchetype = archetype;
        }
    }
}

// == phys::CandidateCollision (physics.hpp)
struct OverlapRow {
    u32 aArch; i32 aRow;
    u32 bArch; i32 bRow;
    u32 aPrim, bPrim;
};

// One warp per world: candidate i of world w -> row worldOffsets[w] + i.  Side a is the
// iterating body (smaller entity ID) again and the primitive indices are those within each
// body (Candidate::pad[0]); column 0 is Entity {0, 0} as Context::makeTemporary writes it.
__global__ void __launch_bounds__(kPhysWorldThreads)
physEmitOverlapsKernel(EngineState *Sp, u32 archetype, i32 col)
{
    const EngineState &S = *Sp;
    const PhysicsState &P = *S.physics;
    const i32 w = (i32)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (w >= (i32)S.numWorlds) return;
    const TableDesc &t = S.tables[archetype];
    const i32 off = t.worldOffsets[w], n = t.worldCounts[w];
    const Candidate *cands = P.candidates + (size_t)w * P.maxCandidatesPerWorld;
    u64 *entities = (u64 *)t.columns[0];
    i32 *worlds = (i32 *)t.columns[1];
    OverlapRow *rows = (OverlapRow *)t.columns[col];
    for (i32 i = lane; i < n; i += 32) {
        const Candidate c = cands[i];
        const u32 rel = c.pad[0];
        const u32 arch0 = c.arch & 0xffu, arch1 = (c.arch >> 8) & 0xffu;
        const bool swapped = (rel >> 16) & 1u;
        OverlapRow r;
        r.aArch = swapped ? arch1 : arch0;
        r.aRow = swapped ? c.bRow : c.aRow;
        r.bArch = swapped ? arch0 : arch1;
        r.bRow = swapped ? c.aRow : c.bRow;
        r.aPrim = rel & 0xffu;
        r.bPrim = (rel >> 8) & 0xffu;
        entities[off + i] = 0ull;
        worlds[off + i] = w;
        rows[off + i] = r;
    }
}

// =============================================================================================
// Host side
// =============================================================================================

bool physicsHostCreate(Executor *ex, std::string *err)
{
    PhysicsHost *ph = new PhysicsHost();
    ex->physics = ph;
    memset(&ph->hPhys, 0, sizeof(PhysicsState));
    if (cudaMalloc((void **)&ph->dPhys, sizeof(PhysicsState)) != cudaSuccess) {
        *err = "physics state allocation failed";
        return false;
    }
    ex->allocations.push_back(ph->dPhys);
    cudaMemset(ph->dPhys, 0, sizeof(PhysicsState));
    ex->hState->physics = ph->dPhys;
    return true;
}

static size_t largeStageBytes(int max_hull_size)
{
    return (size_t)kLargeWarps * max_hull_size * kLargeStageBytesPerEntry;
}

bool physicsHostAfterRegistry(Executor *ex, std::string *err)
{
    PhysicsHost *ph = ex->physics;
    EngineState &S = *ex->hState;
    cudaMemcpy(&ph->hPhys, ph->dPhys, sizeof(PhysicsState), cudaMemcpyDeviceToHost);
    PhysicsState &P = ph->hPhys;
    if (!P.registered) return true;   // simulator without physics
    ph->active = true;

    // archetypes that carry the whole RigidBody bundle, ascending id == the
    // CPU backend's query iteration order
    P.numBodyArchetypes = 0;
    memset(P.bodyIndex, 0xff, sizeof(P.bodyIndex));
    for (uint32_t a = 0; a < S.numArchetypes; a++) {
        if (!S.archetypes[a].registered) continue;
        BodyArchetype b;
        b.archetype = a;
        bool all = true;
        for (int pc = 0; pc < PCCount; pc++) {
            int col = S.columnLookup[a][P.componentIDs[pc]];
            // TGS keeps no per-body solver state (its RigidBody bundle ends at ExternalTorque)
            const bool solver_state = pc == PCPrevState || pc == PCPreSolvePos || pc == PCPreSolveVel;
            if (col < 0 && !(solver_state && P.solver == 1u)) { all = false; break; }
            b.cols[pc] = col;
        }
        if (!all) continue;
        if (P.numBodyArchetypes >= (uint32_t)kMaxBodyArchetypes) {
            *err = "too many rigid-body archetypes";
            return false;
        }
        P.bodyIndex[a] = (signed char)P.numBodyArchetypes;
        P.bodies[P.numBodyArchetypes++] = b;
    }
    P.jointCol = S.columnLookup[P.jointArchetype][P.cidJointConstraint];

    P.maxCandidatesPerWorld = (i32)ex->knobs.maxCandidatesPerWorld;
    P.maxContactsPerWorld = (i32)ex->knobs.maxContactsPerWorld;
    const size_t W = S.numWorlds;
    auto alloc = [&](void **p, size_t bytes) {
        if (cudaMalloc(p, bytes) != cudaSuccess) return false;
        ex->allocations.push_back(*p);
        cudaMemset(*p, 0, bytes);
        return true;
    };
    // The step's work lists.  Their counters are one array, hull - hull, other, large pairs,
    // large worlds, so one memset before the candidate search resets the lists a step uses.
    PairListCounters *pair_counters = nullptr;
    auto alloc_list = [&](PairList &list, int k) {
        list.counters = pair_counters + k;
        return alloc((void **)&list.entries, sizeof(PairEntry) * W * P.maxCandidatesPerWorld);
    };
    if (!alloc((void **)&P.candidates, sizeof(Candidate) * W * P.maxCandidatesPerWorld) ||
        !alloc((void **)&P.candCounts, sizeof(i32) * W) ||
        !alloc((void **)&P.contacts, sizeof(Contact) * W * P.maxCandidatesPerWorld) ||
        !alloc((void **)&P.candHit, sizeof(i32) * W * P.maxCandidatesPerWorld) ||
        !alloc((void **)&P.contactOrder, sizeof(i32) * W * P.maxContactsPerWorld) ||
        !alloc((void **)&pair_counters, sizeof(PairListCounters) * 4) ||
        !alloc_list(P.hullPairs, 0) ||
        !alloc_list(P.otherPairs, 1) ||
        !alloc((void **)&P.contactCounts, sizeof(i32) * W) ||
        !alloc((void **)&P.contactMaxLevel, sizeof(i32) * W)) {
        *err = "physics buffers allocation failed";
        return false;
    }
    // hulls past the staging caps: the third work list and its kernel's shared memory
    const int max_hull_size = (int)ex->knobs.maxHullSize;
    P.maxHullSize = max_hull_size;
    if (max_hull_size > kMinHullSizeCap) {
        if (!alloc_list(P.largePairs, 2) ||
            !alloc((void **)&ph->classInfo, sizeof(i32) * 3)) {
            *err = "physics buffers allocation failed";
            return false;
        }
        if (cudaFuncSetAttribute(physNarrowphaseLargeKernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)largeStageBytes(max_hull_size)) != cudaSuccess) {
            cudaGetLastError();
            *err = "the large-hull narrowphase's shared memory (MADRONA_B200_MAX_HULL_SIZE) does not fit the device";
            return false;
        }
    }
    // worlds past 128 bodies: their work list and the global contact level table (4 bytes per
    // world and body slot)
    const int max_world_bodies = (int)ex->knobs.maxWorldBodies;
    P.maxWorldBodies = max_world_bodies;
    if (max_world_bodies > kMinWorldBodiesCap) {
        P.largeWorlds.counters = pair_counters + 3;
        if (!alloc((void **)&P.largeWorlds.entries, sizeof(PairEntry) * W) ||
            !alloc((void **)&P.levelScratch, sizeof(i32) * W * max_world_bodies)) {
            *err = "physics buffers allocation failed";
            return false;
        }
    }
    cudaMemcpy(ph->dPhys, &P, sizeof(PhysicsState), cudaMemcpyHostToDevice);
    // the position solve's body stage, and L1 for the rest (see kPosSolveCarveoutPercent)
    if (cudaFuncSetAttribute(physSolvePositionsKernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                             kPosSolveCarveoutPercent) != cudaSuccess) {
        *err = "setting the position solve's shared-memory carveout failed";
        return false;
    }
    return true;
}

// MADRONA_B200_MAX_HULL_SIZE > 16: class of every primitive the worlds' bodies can refer to,
// from the ObjectManager as it is now (like the sphere flag above: build the launch graph
// after the ObjectManager is final).  Without a large primitive the table stays unset and
// the step is captured exactly as without the knob.
static void physicsClassifyPrims(Executor *ex)
{
    PhysicsHost *ph = ex->physics;
    PhysicsState &P = ph->hPhys;
    ph->largeHulls = false;
    ph->largeError.clear();
    if (P.maxHullSize <= kMinHullSizeCap) return;
    auto fail = [&](const char *what) {
        cudaGetLastError();
        ph->largeError = what;
    };
    i32 info[3] = { 0, 0, 0 };
    cudaMemset(ph->classInfo, 0, sizeof(info));
    physPrimExtentKernel<<<ex->numSMs * 4, 256>>>(ex->dState, ph->classInfo);
    if (cudaMemcpy(info, ph->classInfo, sizeof(info), cudaMemcpyDeviceToHost) != cudaSuccess) {
        return fail("classifying the collision primitives failed");
    }
    if (info[1] != 0) {
        return fail("MADRONA_B200_MAX_HULL_SIZE needs one ObjectManager shared by all worlds");
    }
    const i32 num_prims = info[0];
    if (num_prims > ph->primClassCapacity) {
        void *table = nullptr;
        if (cudaMalloc(&table, (size_t)num_prims) != cudaSuccess) return fail("primitive class table allocation failed");
        ex->allocations.push_back(table);
        ph->primClass = (unsigned char *)table;
        ph->primClassCapacity = num_prims;
    }
    if (num_prims > 0) {
        physClassifyPrimsKernel<<<(num_prims + 255) / 256, 256>>>(ex->dState, ph->primClass, num_prims, ph->classInfo);
        if (cudaMemcpy(info, ph->classInfo, sizeof(info), cudaMemcpyDeviceToHost) != cudaSuccess) {
            return fail("classifying the collision primitives failed");
        }
    }
    ph->largeHulls = info[2] != 0;
    P.primClass = ph->largeHulls ? ph->primClass : nullptr;
    P.numPrimClasses = ph->largeHulls ? num_prims : 0;
    cudaMemcpy(&ph->dPhys->primClass, &P.primClass, sizeof(P.primClass), cudaMemcpyHostToDevice);
    cudaMemcpy(&ph->dPhys->numPrimClasses, &P.numPrimClasses, sizeof(P.numPrimClasses), cudaMemcpyHostToDevice);
    if (!ph->largeHulls) return;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, physNarrowphaseLargeKernel, kLargeThreads,
                                                      largeStageBytes(P.maxHullSize)) != cudaSuccess) {
        cudaGetLastError();
        per_sm = 0;
    }
    ph->largeBlocks = (unsigned)ex->numSMs * (unsigned)per_sm;
}

void physicsBeforeGraphCapture(Executor *ex)
{
    PhysicsHost *ph = ex->physics;
    if (!ph || !ph->active) return;
    u32 flag = 0;
    cudaMemcpy(&flag, &ph->dPhys->hasSpherePrims, sizeof(u32), cudaMemcpyDeviceToHost);
    ph->spheres = flag != 0;
    // the narrowphase grid is exactly what is resident at once
    int per_sm = 0;
    const cudaError_t e = ph->spheres
        ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, physNarrowphaseKernel<true>, kNarrowThreads, 0)
        : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, physNarrowphaseKernel<false>, kNarrowThreads, 0);
    if (e != cudaSuccess) cudaGetLastError();
    ph->narrowBlocks = e == cudaSuccess ? (unsigned)ex->numSMs * (unsigned)per_sm : 0u;
    if (ph->hPhys.maxWorldBodies > kMinWorldBodiesCap) {
        per_sm = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, physFindCandidatesLargeKernel,
                                                          kLargeSearchThreads, 0) != cudaSuccess) {
            cudaGetLastError();
            per_sm = 0;
        }
        ph->largeSearchBlocks = (unsigned)ex->numSMs * (unsigned)per_sm;
    }
    physicsClassifyPrims(ex);
}

const PhysicsState *physicsHostState(Executor *ex)
{
    const PhysicsHost *ph = ex->physics;
    return ph && ph->active ? &ph->hPhys : nullptr;
}

void physicsHostDestroy(Executor *ex)
{
    delete ex->physics;
    ex->physics = nullptr;
}

static dim3 bodyGrid(Executor *ex)
{
    const PhysicsState &P = ex->physics->hPhys;
    int max_cap = 256;
    for (uint32_t i = 0; i < P.numBodyArchetypes; i++) {
        max_cap = std::max(max_cap, ex->hState->tables[P.bodies[i].archetype].capacity);
    }
    int blocks = std::min((max_cap + 255) / 256, ex->numSMs * 4);
    return dim3((unsigned)std::max(blocks, 1), std::max(P.numBodyArchetypes, 1u));
}

// Lanes per world of the velocity solve: 16 while the worlds fit one wave of the
// 16-lane kernel (kVelSolveBlocksPerSM blocks of 4 worlds per SM), else 8.  Fewer
// lanes per world spread a level's contacts over fewer lanes but double the worlds
// resident at once.
static unsigned velocitySolveLanes(const Executor *ex, unsigned W)
{
    const unsigned wide_worlds = (unsigned)ex->numSMs * kVelSolveBlocksPerSM * (kPhysWorldThreads / 16);
    return W <= wide_worlds ? 16u : 8u;
}

bool physicsEnqueueNodes(Executor *ex, const NodeRecord *recs, uint32_t count, cudaStream_t s,
                         std::string *err)
{
    PhysicsHost *ph = ex->physics;
    if (!ph || !ph->active) {
        *err = "physics task recorded but PhysicsSystem::registerTypes was never called";
        return false;
    }
    if (!ph->largeError.empty()) {
        *err = ph->largeError;
        return false;
    }
    EngineState *d = ex->dState;
    const unsigned W = ex->hState->numWorlds;
    const unsigned wgrid = (W + kPhysWarps - 1) / kPhysWarps;
    const unsigned wblock = kPhysWorldThreads;
    const unsigned pos_grid = (W + wblock / kPosSolverLanes - 1) / (wblock / kPosSolverLanes);
    const unsigned vel_lanes = velocitySolveLanes(ex, W);
    const unsigned vel_grid = (W + wblock / vel_lanes - 1) / (wblock / vel_lanes);
    const dim3 bgrid = bodyGrid(ex);
    const bool large_worlds = ph->hPhys.maxWorldBodies > kMinWorldBodiesCap;
    for (uint32_t i = 0; i < count; i++) {
        const NodeRecord &rec = recs[i];
        switch (rec.kind) {
        case NodePhysBroadphaseUpdate:
            // tag 0 (post-integration) never rebuilds in the reference either; a
            // pending rebuild request then simply waits for the next tag-1 node,
            // and the un-refitted leaves are refitted by that rebuild
            physBodyKernel<PhaseUpdateLeaves><<<bgrid, 256, 0, s>>>(d);
            if (rec.userTag == 1) physRebuildKernel<<<(W + 127) / 128, 128, 0, s>>>(d);
            break;
        case NodePhysFindCandidates:
            // joints are iterated per world by the solver: keep their table in
            // world order (the reference sorts Joint here too, xpbd.cpp:1092-1096).
            // Tag 1: the standalone overlap tasks, no solver reads the joints.
            if (rec.userTag != 1) launchSortArchetype(ex, ph->hPhys.jointArchetype, 1, s);
            // the search appends the step's pairs to empty lists: hull - hull, other and, with
            // a hull past the staging caps, large; with worlds past 128 bodies also the list
            // of those worlds (tickets are zero between launches)
            cudaMemsetAsync(ph->hPhys.hullPairs.counters, 0,
                            (large_worlds ? 4 : ph->largeHulls ? 3 : 2) * sizeof(PairListCounters), s);
            physFindCandidatesKernel<<<wgrid, wblock, 0, s>>>(d);
            if (large_worlds) {
                if (ph->largeSearchBlocks == 0) {
                    *err = "large-world candidate search occupancy query failed";
                    return false;
                }
                physFindCandidatesLargeKernel<<<ph->largeSearchBlocks, kLargeSearchThreads, 0, s>>>(d);
            }
            break;
        case NodePhysSubstepBegin:
            physBodyKernel<PhaseIntegrate><<<bgrid, 256, 0, s>>>(d);
            break;
        case NodePhysNarrowphase:
            if (ph->narrowBlocks == 0) {
                *err = "narrowphase occupancy query failed";
                return false;
            }
            if (ph->spheres) physNarrowphaseKernel<true><<<ph->narrowBlocks, kNarrowThreads, 0, s>>>(d);
            else physNarrowphaseKernel<false><<<ph->narrowBlocks, kNarrowThreads, 0, s>>>(d);
            if (ph->largeHulls) {
                if (ph->largeBlocks == 0) {
                    *err = "large-hull narrowphase occupancy query failed";
                    return false;
                }
                physNarrowphaseLargeKernel<<<ph->largeBlocks, kLargeThreads,
                                             largeStageBytes(ph->hPhys.maxHullSize), s>>>(d);
            }
            break;
        case NodePhysSolvePositions:
            physSolvePositionsKernel<<<pos_grid, wblock, 0, s>>>(d);
            break;
        case NodePhysTGSVelocities:
            physBodyKernel<PhaseTGSVelocities><<<bgrid, 256, 0, s>>>(d);
            break;
        case NodePhysTGSPositions:
            physBodyKernel<PhaseTGSPositions><<<bgrid, 256, 0, s>>>(d);
            break;
        case NodePhysSetVelocities:
            physBodyKernel<PhaseSetVelocities><<<bgrid, 256, 0, s>>>(d);
            break;
        case NodePhysSolveVelocities:
            if (vel_lanes == 16) physSolveVelocitiesKernel<16><<<vel_grid, wblock, 0, s>>>(d);
            else physSolveVelocitiesKernel<8><<<vel_grid, wblock, 0, s>>>(d);
            break;
        case NodePhysEmitOverlaps: {
            const EngineState &S = *ex->hState;
            const i32 col = (rec.archetype < S.numArchetypes && rec.component < S.numComponents)
                ? S.columnLookup[rec.archetype][rec.component] : -1;
            if (col < 2) {
                *err = "standalone overlap node: the CandidateTemporary archetype lacks CandidateCollision";
                return false;
            }
            physEmitOverlapsScanKernel<<<1, kEmitScanThreads, 0, s>>>(d, rec.archetype);
            physEmitOverlapsKernel<<<wgrid, wblock, 0, s>>>(d, rec.archetype, col);
            break;
        }
        default:
            *err = "unknown physics node kind " + std::to_string(rec.kind);
            return false;
        }
    }
    return true;
}

uint64_t physicsNodeBytes(Executor *ex, const NodeRecord &rec, const char **name, int64_t *rows)
{
    // SURVEY.md 8(d) algorithmic bytes per unit
    PhysicsHost *ph = ex->physics;
    *rows = 0;
    *name = "physics";
    if (!ph || !ph->active) return 0;
    const PhysicsState &P = ph->hPhys;
    const unsigned W = ex->hState->numWorlds;

    int64_t bodies = 0;
    std::vector<TableDesc> tables(ex->hState->numArchetypes);
    cudaMemcpy(tables.data(), ex->dState->tables, sizeof(TableDesc) * tables.size(), cudaMemcpyDeviceToHost);
    for (uint32_t i = 0; i < P.numBodyArchetypes; i++) bodies += tables[P.bodies[i].archetype].numRows;
    std::vector<i32> counts(W);
    auto total = [&](const i32 *dptr) {
        cudaMemcpy(counts.data(), dptr, sizeof(i32) * W, cudaMemcpyDeviceToHost);
        int64_t t = 0;
        for (i32 c : counts) t += c;
        return t;
    };
    switch (rec.kind) {
    case NodePhysBroadphaseUpdate: *name = "phys_broadphase_update"; *rows = bodies; return 136ull * bodies;
    case NodePhysFindCandidates: *name = "phys_find_candidates"; *rows = total(P.candCounts);
        return 24ull * (*rows) + 40ull * bodies;
    case NodePhysSubstepBegin: *name = "phys_substep"; *rows = bodies; return 192ull * bodies;
    case NodePhysNarrowphase: {
        *name = "phys_narrowphase";
        int64_t q = total(P.candCounts), k = total(P.contactCounts);
        *rows = q;
        return 24ull * q + 88ull * q + 96ull * k;
    }
    case NodePhysSolvePositions: *name = "phys_solve_positions"; *rows = total(P.contactCounts);
        return 368ull * (*rows);
    case NodePhysTGSVelocities: *name = "phys_tgs_velocities"; *rows = bodies; return 104ull * bodies;
    case NodePhysTGSPositions: *name = "phys_tgs_positions"; *rows = bodies; return 80ull * bodies;
    case NodePhysSetVelocities: *name = "phys_set_velocities"; *rows = bodies; return 80ull * bodies;
    case NodePhysSolveVelocities: *name = "phys_solve_velocities"; *rows = total(P.contactCounts);
        return 360ull * (*rows);
    // candidate counts read twice + offsets / counts written, 32 B candidate in, 36 B row out
    case NodePhysEmitOverlaps: *name = "phys_emit_overlaps"; *rows = total(P.candCounts);
        return 68ull * (*rows) + 16ull * W;
    default: return 0;
    }
}

}
