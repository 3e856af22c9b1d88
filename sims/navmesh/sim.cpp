#include "sim.hpp"

#include <cfloat>
#include <cstring>

#ifdef MADRONA_GPU_MODE
#include <madrona/mw_gpu_entry.hpp>
#endif

using namespace madrona;
using namespace madrona::math;

namespace navmesh {

static inline uint32_t fbits(float f)
{
    uint32_t u;
    memcpy(&u, &f, sizeof(u));
    return u;
}

static inline uint32_t hashIn(uint32_t h, uint32_t v)
{
    return utils::int32Hash(h ^ v) + 0x9E3779B9u;
}

static inline uint32_t hashVec(uint32_t h, Vector3 v)
{
    h = hashIn(h, fbits(v.x));
    h = hashIn(h, fbits(v.y));
    return hashIn(h, fbits(v.z));
}

// hash of a navmesh's four arrays
static uint32_t meshHash(const Navmesh &m)
{
    uint32_t h = hashIn(0x2545F491u, m.numVerts);
    h = hashIn(h, m.numTris);
    for (uint32_t i = 0; i < m.numVerts; i++) {
        h = hashVec(h, m.vertices[i]);
    }
    for (uint32_t i = 0; i < 3 * m.numTris; i++) {
        h = hashIn(h, m.triIndices[i]);
        h = hashIn(h, m.triAdjacency[i]);
    }
    for (uint32_t i = 0; i < m.numTris; i++) {
        h = hashIn(h, fbits(m.triSampleAliasTable[i].tau));
        h = hashIn(h, m.triSampleAliasTable[i].alias);
    }
    return h;
}

static inline Navmesh &meshOf(Sim &sim, const AgentInfo &info)
{
    return ((info.idx & 1) || !(sim.flags & FlagPerWorldMeshes)) ? sim.shared : sim.own;
}

static inline RandKey nextKey(Sim &sim, AgentInfo &info)
{
    return rand::split_i(rand::initKey(sim.seed, info.idx), info.samples++);
}

static inline void spawnAgent(Sim &sim, Navmesh &mesh, AgentInfo &info, NavPos &pos, NavPoly &poly,
                              NavGoal &goal)
{
    pos.p = mesh.samplePointAndPoly(nextKey(sim, info), &poly.tri);
    goal.p = mesh.samplePointAndPoly(nextKey(sim, info), &goal.tri);
}

inline void episodeSystem(Engine &ctx, EpisodeState &ep)
{
    ep.respawn = 0;
    ep.step += 1;
    if (ep.step >= ctx.data().episodeLen) {
        ep.step = 0;
        ep.episode += 1;
        ep.respawn = 1;
    }
}

// Dijkstra field from the goal: the agent's distance to its goal and its next waypoint
inline void dijkstraSystem(Engine &ctx, NavPos &pos, NavPoly &poly, NavGoal &goal, NavDist &dist,
                           Waypoint &wp, DijkstraStats &stats, AgentInfo &info)
{
    Sim &sim = ctx.data();
    Navmesh &mesh = meshOf(sim, info);
    stats = DijkstraStats { 0, 0 };
    wp = Waypoint { pos.p, poly.tri };
    dist.d = FLT_MAX;
    const uint32_t T = mesh.numTris;
    if (T == 0) {
        return;
    }
    float *d = (float *)ctx.tmpAlloc(sizeof(float) * T);
    Vector3 *entry = (Vector3 *)ctx.tmpAlloc(sizeof(Vector3) * T);
    uint32_t *heap = (uint32_t *)ctx.tmpAlloc(sizeof(uint32_t) * T);
    uint32_t *heap_idx = (uint32_t *)ctx.tmpAlloc(sizeof(uint32_t) * T);
    if (!d || !entry || !heap || !heap_idx) {
        return;
    }

    uint32_t visits = 0, h = 0x811C9DC5u;
    mesh.dijkstrasFromPoly(goal.tri, goal.p, Navmesh::DijkstrasState { d, entry, heap, heap_idx },
        [&](uint32_t tri, Vector3 at, float dd) {
            visits += 1;
            h = hashIn(h, tri);
            h = hashIn(h, fbits(dd));
            h = hashVec(h, at);
        });
    stats = DijkstraStats { visits, h };

    const uint32_t p = poly.tri;
    if (d[p] == FLT_MAX) {
        return;
    }
    if (p == goal.tri) {
        wp = Waypoint { goal.p, p };
        dist.d = pos.p.distance(goal.p);
        return;
    }
    uint32_t next = p;
    float best = d[p];
    for (uint32_t i = 0; i < 3; i++) {
        const uint32_t n = mesh.triAdjacency[3 * p + i];
        if (n != Navmesh::sentinel && d[n] < best) {
            best = d[n];
            next = n;
        }
    }
    wp = Waypoint { entry[p], next };
    dist.d = d[p] + pos.p.distance(entry[p]);
}

// breadth-first search from the agent's triangle; the predicate rejects every fifth
// triangle (by index, shifting with the episode and the agent)
inline void bfsSystem(Engine &ctx, NavPoly &poly, BfsStats &stats, AgentInfo &info)
{
    Sim &sim = ctx.data();
    Navmesh &mesh = meshOf(sim, info);
    stats = BfsStats { 0, 0 };
    const uint32_t T = mesh.numTris;
    if (T == 0) {
        return;
    }
    uint32_t *queue = (uint32_t *)ctx.tmpAlloc(sizeof(uint32_t) * T);
    bool *visited = (bool *)ctx.tmpAlloc(sizeof(bool) * T);
    if (!queue || !visited) {
        return;
    }
    const uint32_t shift = ctx.singleton<EpisodeState>().episode + info.idx;
    const uint32_t start = poly.tri;
    uint32_t accepted = 0, rejected = 0;
    mesh.bfsFromPoly(start, Navmesh::BFSState { queue, visited }, [&](uint32_t tri) {
        if (tri != start && (tri + shift) % 5 == 0) {
            rejected += 1;
            return false;
        }
        accepted += 1;
        return true;
    });
    stats = BfsStats { accepted, rejected };
}

inline void moveSystem(Engine &ctx, NavPos &pos, NavPoly &poly, NavGoal &goal, Waypoint &wp,
                       AgentInfo &info)
{
    Sim &sim = ctx.data();
    Navmesh &mesh = meshOf(sim, info);
    if (mesh.numTris == 0) {
        return;
    }
    if (ctx.singleton<EpisodeState>().respawn) {
        spawnAgent(sim, mesh, info, pos, poly, goal);
        return;
    }
    const Vector3 delta = wp.p - pos.p;
    const float len = delta.length();
    if (len <= kAgentSpeed) {
        const bool at_goal = poly.tri == goal.tri;
        pos.p = wp.p;
        poly.tri = wp.nextTri;
        if (at_goal) {
            info.reached += 1;
            goal.p = mesh.samplePointAndPoly(nextKey(sim, info), &goal.tri);
        }
    } else {
        pos.p = pos.p + delta * (kAgentSpeed / len);
    }
}

void Sim::registerTypes(ECSRegistry &registry, const Config &)
{
    registry.registerComponent<NavPos>();
    registry.registerComponent<NavPoly>();
    registry.registerComponent<NavGoal>();
    registry.registerComponent<NavDist>();
    registry.registerComponent<Waypoint>();
    registry.registerComponent<DijkstraStats>();
    registry.registerComponent<BfsStats>();
    registry.registerComponent<AgentInfo>();
    registry.registerComponent<LandmarkID>();
    registry.registerSingleton<MeshInfo>();
    registry.registerSingleton<EpisodeState>();

    registry.registerArchetype<Agent>(ComponentMetadataSelector<> {}, ArchetypeFlags::None, kNumAgents);
    registry.registerArchetype<Landmark>();

    registry.exportColumn<Agent, NavPos>((uint32_t)ExportID::AgentPos);
    registry.exportColumn<Agent, NavPoly>((uint32_t)ExportID::AgentPoly);
    registry.exportColumn<Agent, NavDist>((uint32_t)ExportID::AgentDist);
    registry.exportColumn<Agent, DijkstraStats>((uint32_t)ExportID::DijkstraStats);
    registry.exportColumn<Agent, BfsStats>((uint32_t)ExportID::BfsStats);
    registry.exportColumn<Agent, NavGoal>((uint32_t)ExportID::GoalPos);
    registry.exportSingleton<MeshInfo>((uint32_t)ExportID::MeshInfo);
}

void Sim::setupTasks(TaskGraphManager &mgr, const Config &)
{
    TaskGraphBuilder &b = mgr.init(TaskGraphID::Step);
    auto reset = b.addToGraph<ResetTmpAllocNode>({});
    auto episode = b.addToGraph<ParallelForNode<Engine, episodeSystem, EpisodeState>>({ reset });
    auto dijkstra = b.addToGraph<ParallelForNode<Engine, dijkstraSystem,
        NavPos, NavPoly, NavGoal, NavDist, Waypoint, DijkstraStats, AgentInfo>>({ episode });
    auto bfs = b.addToGraph<ParallelForNode<Engine, bfsSystem, NavPoly, BfsStats, AgentInfo>>({ dijkstra });
    b.addToGraph<ParallelForNode<Engine, moveSystem, NavPos, NavPoly, NavGoal, Waypoint, AgentInfo>>({ bfs });
}

Sim::Sim(Engine &ctx, const Config &cfg, const WorldInit &init)
    : WorldBase(ctx),
      own { nullptr, nullptr, nullptr, nullptr, 0, 0 },
      shared(cfg.shared),
      seed(init.seed),
      episodeLen(cfg.episodeLen),
      flags(cfg.flags)
{
    MeshInfo info {};
    if (flags & FlagPerWorldMeshes) {
        Plan *plan = (Plan *)ctx.tmpAlloc(sizeof(Plan));
        if (plan) {
            makePlan(seed, (flags & FlagBadPolygon) && ctx.worldID().idx == 1, *plan);
            own = Navmesh::initFromPolygons((Vector3 *)plan->xyz, plan->idxs, plan->offsets, plan->sizes,
                                            plan->numVerts, plan->numPolys);
            for (uint32_t i = 0; i < plan->numPolys; i++) {
                Entity e = ctx.makeEntity<Landmark>();
                ctx.get<LandmarkID>(e).poly = i;
            }
        }
        info.v[0] = own.numTris ? meshHash(own) : 0;
        info.v[1] = own.numTris;
        info.v[2] = own.numVerts;
    }
    info.v[3] = meshHash(shared);
    info.v[4] = shared.numTris;
    ctx.singleton<MeshInfo>() = info;
    ctx.singleton<EpisodeState>() = EpisodeState { 0, 0, 0, 0 };

    for (int32_t i = 0; i < kNumAgents; i++) {
        Entity e = ctx.makeEntity<Agent>();
        agents[i] = e;
        AgentInfo &ai = ctx.get<AgentInfo>(e);
        ai = AgentInfo { (uint32_t)i, 0, 0, 0 };
        NavPos &pos = ctx.get<NavPos>(e);
        NavPoly &poly = ctx.get<NavPoly>(e);
        NavGoal &goal = ctx.get<NavGoal>(e);
        pos.p = Vector3 { 0.f, 0.f, 0.f };
        poly.tri = Navmesh::sentinel;
        goal = NavGoal { Vector3 { 0.f, 0.f, 0.f }, Navmesh::sentinel };
        ctx.get<NavDist>(e).d = FLT_MAX;
        ctx.get<Waypoint>(e) = Waypoint { Vector3 { 0.f, 0.f, 0.f }, Navmesh::sentinel };
        ctx.get<DijkstraStats>(e) = DijkstraStats { 0, 0 };
        ctx.get<BfsStats>(e) = BfsStats { 0, 0 };
        Navmesh &mesh = meshOf(*this, ai);
        if (mesh.numTris != 0) {
            spawnAgent(*this, mesh, ai, pos, poly, goal);
        }
    }
}

}

#ifdef MADRONA_GPU_MODE
MADRONA_BUILD_MWGPU_ENTRY(navmesh::Engine, navmesh::Sim, navmesh::Config, navmesh::WorldInit);
#endif
