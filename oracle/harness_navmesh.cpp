// TEST INFRASTRUCTURE ONLY: sims/navmesh on the reference CPU backend.  The navmesh every
// world shares is built here with the reference's host Navmesh::initFromPolygons (the GPU
// engine builds it with mb2_navmesh_create).  Built by oracle/navmesh.mk.
#include <madrona/mw_cpu.hpp>
#include "../sims/navmesh/sim.hpp"
#include "harness.hpp"

using namespace navmesh;

int main(int argc, char **argv)
{
    oracle::Args args = oracle::parseArgs(argc, argv);
    static Plan plan;
    makePlan(kSharedPlanSeed, 0, plan);
    Config cfg {};
    cfg.shared = madrona::Navmesh::initFromPolygons((madrona::math::Vector3 *)plan.xyz, plan.idxs,
        plan.offsets, plan.sizes, plan.numVerts, plan.numPolys);
    cfg.episodeLen = (uint32_t)(args.extra[0] ? args.extra[0] : 40);
    cfg.flags = args.extra[2] ? (uint32_t)FlagPerWorldMeshes : 0u;
    std::vector<WorldInit> inits(args.numWorlds);
    for (int64_t i = 0; i < args.numWorlds; i++) {
        inits[i].seed = (uint32_t)(args.extra[1] + i);
    }

    using Exec = madrona::TaskGraphExecutor<Engine, Sim, Config, WorldInit>;
    Exec exec({
        .numWorlds = (uint32_t)args.numWorlds,
        .numExportedBuffers = (uint32_t)ExportID::NumExports,
        .numWorkers = (uint32_t)args.numWorkers,
    }, cfg, inits.data(), (madrona::CountT)TaskGraphID::NumTaskGraphs);

    const size_t W = (size_t)args.numWorlds, A = (size_t)kNumAgents;
    return oracle::runTrace(exec, args, {},
        { { (int)ExportID::AgentPos, [=] { return W * A * 12; } },
          { (int)ExportID::AgentPoly, [=] { return W * A * 4; } },
          { (int)ExportID::AgentDist, [=] { return W * A * 4; } },
          { (int)ExportID::DijkstraStats, [=] { return W * A * 8; } },
          { (int)ExportID::BfsStats, [=] { return W * A * 8; } },
          { (int)ExportID::GoalPos, [=] { return W * A * 16; } },
          { (int)ExportID::MeshInfo, [=] { return W * sizeof(MeshInfo); } } });
}
