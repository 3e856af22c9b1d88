// Fixture simulator for navigation meshes (<madrona/navmesh.hpp>).  ECS only.
//
// Every world builds its own navmesh in its constructor with Navmesh::initFromPolygons,
// from a seeded floor plan (plan.hpp), and all worlds share one more navmesh passed in
// Config (built by mb2_navmesh_create on the GPU engine, by the reference's host
// initFromPolygons on the CPU backend).  Agents alternate between the two meshes.  Each
// step, per agent:
//   * DijkstraNode: a Dijkstra field from the agent's goal over its mesh, in tmpAlloc
//     scratch; the agent's next waypoint is the entry point of its triangle, and its
//     distance to the goal is recorded with the visit count and a hash of the visit order;
//   * BfsNode: a breadth-first search from the agent's triangle whose predicate rejects
//     some triangles; it counts what it reaches;
//   * MoveNode: a bounded step towards the waypoint; at the goal a new goal is sampled,
//     and every episodeLen steps all agents respawn (samplePointAndPoly).
// All floats are computed without FMA contraction on both backends, so every exported
// column matches the reference bit for bit.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/rand.hpp>
#include <madrona/navmesh.hpp>
#include <madrona/memory.hpp>

#include "plan.hpp"

namespace navmesh {

using madrona::Entity;
using madrona::CountT;
using madrona::Navmesh;
using madrona::math::Vector3;

constexpr int32_t kNumAgents = 6;
constexpr float kAgentSpeed = 0.4f;

enum class ExportID : uint32_t {
    AgentPos,
    AgentPoly,
    AgentDist,
    DijkstraStats,
    BfsStats,
    GoalPos,
    MeshInfo,
    NumExports,
};

enum class TaskGraphID : uint32_t {
    Step,
    NumTaskGraphs,
};

enum ConfigFlags : uint32_t {
    FlagPerWorldMeshes = 1u << 0,    // else every agent walks the shared mesh
    FlagBadPolygon = 1u << 1,        // world 1's plan has a 2-vertex polygon
};

struct NavPos { Vector3 p; };
struct NavPoly { uint32_t tri; };
struct NavGoal { Vector3 p; uint32_t tri; };
struct NavDist { float d; };
struct Waypoint { Vector3 p; uint32_t nextTri; };
// Dijkstra visits and the hash of (triangle, distance bits, entry-point bits) in visit order
struct DijkstraStats { uint32_t visits; uint32_t hash; };
// BFS triangles accepted and rejected by the predicate
struct BfsStats { uint32_t accepted; uint32_t rejected; };
struct AgentInfo {
    uint32_t idx;          // agent index in its world; odd agents walk the shared mesh
    uint32_t samples;      // random keys drawn so far
    uint32_t reached;      // goals reached
    uint32_t pad;
};

// the world's mesh (hash of its arrays, triangles, vertices) and the shared mesh (hash,
// triangles), as the world constructor saw them
struct MeshInfo { uint32_t v[6]; };
struct EpisodeState { uint32_t step; uint32_t episode; uint32_t respawn; uint32_t pad; };

struct Agent : public madrona::Archetype<
    NavPos, NavPoly, NavGoal, NavDist, Waypoint, DijkstraStats, BfsStats, AgentInfo
> {};

// one per polygon of the world's plan: a dynamic table filled in the constructor
struct LandmarkID { uint32_t poly; };
struct Landmark : public madrona::Archetype<LandmarkID> {};

struct Config {
    Navmesh shared;          // 40 bytes, pointers valid where the simulator runs
    uint32_t episodeLen;
    uint32_t flags;
};

struct WorldInit {
    uint32_t seed;
};

class Engine;

struct Sim : public madrona::WorldBase {
    static void registerTypes(madrona::ECSRegistry &registry, const Config &cfg);
    static void setupTasks(madrona::TaskGraphManager &mgr, const Config &cfg);

    Sim(Engine &ctx, const Config &cfg, const WorldInit &init);

    Navmesh own;
    Navmesh shared;
    uint32_t seed;
    uint32_t episodeLen;
    uint32_t flags;
    Entity agents[kNumAgents];
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
