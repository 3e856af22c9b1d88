// physics_state.h -- layouts shared by the NVRTC-side physics API
// (device/madrona/physics.hpp: what simulator code calls) and the ahead-of-time
// physics kernels (kernels_physics.cu).  Plain structs, no std headers.
//
// The public component structs (Velocity, CollisionPrimitive, ObjectManager,
// RigidBodyMetadata, HalfEdgeMesh ...) keep the reference's field order and
// sizes (include/madrona/physics.hpp:12-153, geo.hpp:7-45) so a simulator's
// ObjectManager blob is interchangeable between the reference CPU backend and
// this engine.  Engine-internal state (candidate / contact buffers, per-world
// BVH storage) is laid out for the GPU instead of being ECS archetypes.
#pragma once

#include "mb2_state.h"

namespace mb2 {

struct PVec3 { float x, y, z; };
struct PQuat { float w, x, y, z; };
struct alignas(16) PVec4 { float x, y, z, w; };
struct PAABB { PVec3 pMin, pMax; };

// == broadphase::BVH::Node (include/madrona/broadphase.hpp:62-78): 4-wide node,
// child boxes in SoA, leaf children tagged with bit 31, sentinel = -1.
struct BVHNode {
    float minX[4];
    float minY[4];
    float minZ[4];
    float maxX[4];
    float maxY[4];
    float maxZ[4];
    i32 children[4];
    i32 parentID;
};

struct LeafTransform {
    PVec3 pos;
    PQuat rot;
    PVec3 scale;
};

// One per world: the payload of the broadphase::BVH singleton component.
struct WorldBVH {
    BVHNode *nodes;
    u64 *leafEntities;        // Entity {gen,id} packed as in the table column
    const void *objMgr;       // const phys::ObjectManager *
    i32 *leafObjIDs;
    PAABB *leafAABBs;
    LeafTransform *leafTransforms;
    u32 *leafParents;         // (node << 2) | child
    i32 *sortedLeaves;
    // Leaves in the order an un-pruned traversal reports them (children 0..3
    // scanned in order, inner children visited LIFO).  Pruning never reorders
    // the survivors, so a query's result list is this list filtered by box
    // overlap -- which lets the candidate search run as a uniform loop.
    i32 *traversalOrder;
    // The same list with the boxes inlined, 32 B per entry: the leaf's slot box in
    // its parent node (grow-only between rebuilds) + the leaf index --
    //   {min.x, min.y, min.z, max.x}, {max.y, max.z, leaf (int bits), 0}
    // kept current by rebuild / refit, read by the candidate search and by
    // BVH::traceRay as a flat, coalesced array (no node pointer chasing).
    PVec4 *orderedBoxes;
    i32 *leafOrderPos;        // leaf -> position in the list
    i32 numNodes;
    i32 numAllocatedNodes;
    i32 numLeaves;
    i32 numAllocatedLeaves;
    float velExpansion;
    float accelExpansion;
    i32 forceRebuild;
    i32 numTraversal;
};

// == phys::PhysicsSystemState (src/physics/physics_impl.hpp:7-15)
struct PhysicsWorldParams {
    float deltaT;
    float h;
    PVec3 g;
    float gMagnitude;
    float restitutionThreshold;
    u32 contactArchetypeID;
    u32 jointArchetypeID;
};

// Class of a candidate pair: the OR of its primitives' types (sphere 1, hull 2, plane 4)
enum PairClass : u32 {
    PairSphereSphere = 1,
    PairHullHull = 2,
    PairSphereHull = 3,
    PairSpherePlane = 5,
    PairHullPlane = 6,
};

// Role of phys::CandidateCollision (physics.hpp:52-57: two Locs + two primitive
// indices, 24 B), resolved by the candidate search into everything about the pair
// that stays fixed for the step, so that every substep's narrowphase only loads the
// poses and the primitive boxes.  Side a / b are already in primitive type order
// (sphere < hull < plane):
//   aPrim, bPrim = indices into the world's ObjectManager::prims
//   arch  = aArch | bArch << 8 | PairClass << 16
//   slots = aSlot | aMutable << 15 | ... same for b in the high half, i.e.
//           ((slot << 1) | mutable) per side with slot = index of the body in
//           its world's body list (0x7fff: unknown) and mutable = "writing the
//           body back can change it" (see rotationIsNormalizeFixpoint).
//   pad[0] = the pair as the reference's CandidateCollision row has it, for the
//           standalone overlap rows (NodePhysEmitOverlaps): aRel | bRel << 8 |
//           swapped << 16, with aRel / bRel the primitive indices within the
//           iterating body (smaller entity ID) and its partner, and swapped set
//           when side a above is the partner (primitive type order reversed it)
struct alignas(16) Candidate {
    u32 aPrim;
    u32 bPrim;
    i32 aRow;
    i32 bRow;
    u32 arch;
    u32 slots;
    u32 pad[2];
};

struct PairEntry {
    i32 world;
    i32 cand;
};

// A work list of the step's pairs, in any order across worlds: appended by the candidate
// search, handed out to the narrowphase's warps by the ticket.
struct PairListCounters {
    i32 count;        // entries, reset before each candidate search
    i32 ticket;       // next work item; zero between launches
    i32 finished;     // warps of the launch that took their last ticket; zero between launches
};

struct PairList {
    PairEntry *entries;          // [numWorlds * maxCandidatesPerWorld]
    PairListCounters *counters;
};

// == phys::ContactConstraint (physics.hpp:59-65) + xpbd::XPBDContactState
struct Contact {
    u32 refArch; i32 refRow;
    u32 altArch; i32 altRow;
    float points[4][4];       // xyz + penetration depth
    i32 numPoints;
    PVec3 normal;
    float lambdaN;            // XPBDContactState::lambdaN[0], the only one ever read (xpbd.cpp:1028)
    u32 refInfo;              // (world body slot << 1) | mutable of ref / alt (Candidate::slots)
    u32 altInfo;
    // Dependency level inside the world's contact list: contacts of one level
    // touch disjoint (mutable) bodies and every earlier contact they could
    // depend on has a lower level, so solving level by level in parallel is
    // bit-identical to the reference's sequential Gauss-Seidel sweep.
    i32 level;
};

enum PhysCol : int {
    PCPosition = 0, PCRotation, PCScale, PCObjectID, PCResponseType, PCLeafID,
    PCVelocity, PCExtForce, PCExtTorque, PCPrevState, PCPreSolvePos, PCPreSolveVel,
    PCCount
};

constexpr int kMaxBodyArchetypes = 16;
constexpr int kMaxHullVerts = 16;     // narrowphase staging caps of the group-per-pair path
constexpr int kMaxHullFaces = 16;
constexpr int kMaxFaceVerts = 8;
// MADRONA_B200_MAX_HULL_SIZE: vertices / faces of a hull the warp-per-pair path stages (the
// reference's narrowphase stages hull - hull pairs in 256-entry halves of its 512-entry arrays)
constexpr int kMinHullSizeCap = kMaxHullVerts;
constexpr int kMaxHullSizeCap = 255;

// PhysicsState::primClass: which narrowphase path a collision primitive takes
enum PrimClass : unsigned char {
    PrimSmall = 0,      // sphere, plane, or a hull within the three staging caps above
    PrimLarge = 1,      // a hull within PhysicsState::maxHullSize vertices and faces
    PrimTooLarge = 2,   // a hull past it: the pair raises ErrPhysicsOverflow
};
constexpr int kMaxLevelBodies = 128;  // bodies per world tracked by the contact level scan in shared memory
// MADRONA_B200_MAX_BODIES_PER_WORLD: BVH leaves (rigid bodies) a world may hold.  Worlds of
// up to kMinWorldBodiesCap leaves take the warp-per-world candidate search and the shared
// level table; larger ones, up to the knob, the block-per-world search and a global table.
constexpr int kMinWorldBodiesCap = 128;
constexpr int kMaxWorldBodiesCap = 4096;

struct BodyArchetype {
    u32 archetype;
    i32 cols[PCCount];
};

struct PhysicsState {
    // ---- written by the device-side PhysicsSystem::registerTypes (1 thread)
    u32 registered;
    u32 solver;
    u32 componentIDs[PCCount];
    u32 cidJointConstraint;
    u32 bvhArchetype;            // singleton archetypes
    u32 paramsArchetype;
    u32 objectDataArchetype;
    u32 jointArchetype;
    // set by PhysicsSystem::registerEntity when an object with a sphere primitive
    // joins a world: selects the narrowphase kernel that carries the sphere-hull
    // (GJK) path
    u32 hasSpherePrims;

    // ---- filled by the host after registerTypes
    u32 numBodyArchetypes;
    BodyArchetype bodies[kMaxBodyArchetypes];   // ascending archetype id
    signed char bodyIndex[kMaxArchetypes];      // archetype id -> index into bodies[] or -1
    i32 jointCol;

    Candidate *candidates;       // [numWorlds][maxCandidatesPerWorld]
    i32 *candCounts;             // [numWorlds]
    i32 maxCandidatesPerWorld;
    // A candidate's contact lives in the slot of the same index (so the dense
    // narrowphase kernels need no per-world ordering); candHit marks the slots
    // that hold a contact this substep, contactOrder lists them in candidate
    // order (== the CPU backend's contact order) for the solvers.
    Contact *contacts;           // [numWorlds][maxCandidatesPerWorld]
    i32 *candHit;                // [numWorlds][maxCandidatesPerWorld]
    i32 *contactOrder;           // [numWorlds][maxContactsPerWorld] -> slot
    i32 *contactCounts;
    i32 *contactMaxLevel;        // [numWorlds]
    i32 maxContactsPerWorld;
    // the step's candidates as two work lists, hull - hull pairs and all other pairs, read
    // by every substep's narrowphase, which hands out the items of both by hullPairs' ticket
    PairList hullPairs;
    PairList otherPairs;

    // ---- hulls past the staging caps (MADRONA_B200_MAX_HULL_SIZE > 16)
    i32 maxHullSize;             // 16: none of the fields below is used
    // One PrimClass per primitive of the worlds' ObjectManager, written before the launch
    // graph is captured; null when no primitive is large (the step then runs exactly the
    // kernels it runs without the knob).  A primitive index past the table (an object
    // first used after the capture) counts as too large.
    const unsigned char *primClass;
    i32 numPrimClasses;
    // the step's pairs with a large or too large primitive, of every pair type: the third
    // work list, read by physNarrowphaseLargeKernel
    PairList largePairs;

    // ---- worlds past 128 bodies (MADRONA_B200_MAX_BODIES_PER_WORLD > 128)
    i32 maxWorldBodies;          // 128: none of the fields below is used
    // the step's worlds with 128 < numTraversal <= maxWorldBodies, PairEntry { world,
    // numTraversal }: appended by physFindCandidatesKernel, searched by
    // physFindCandidatesLargeKernel (one block per world)
    PairList largeWorlds;
    // [numWorlds][maxWorldBodies] per-body contact levels of the worlds with more body
    // slots than the shared table holds (orderContacts)
    i32 *levelScratch;
};

}
