// TEST INFRASTRUCTURE ONLY: sims/triggers on the reference CPU backend (the
// reference's own broadphase, standalone overlap tasks and overlap queries).
// Built by oracle/overlap.mk.
#include <madrona/mw_cpu.hpp>
#include "../sims/triggers/sim.hpp"
#include "harness.hpp"

using namespace triggers;

int main(int argc, char **argv)
{
    oracle::Args args = oracle::parseArgs(argc, argv);
    Config cfg { (madrona::phys::ObjectManager *)oracle::loadObjectsBlob(oracle::objectsPathArg(argc, argv)) };
    std::vector<WorldInit> inits(args.numWorlds);
    for (int64_t i = 0; i < args.numWorlds; i++) inits[i].seed = (uint32_t)(args.extra[0] + i);

    using Exec = madrona::TaskGraphExecutor<Engine, Sim, Config, WorldInit>;
    Exec exec({
        .numWorlds = (uint32_t)args.numWorlds,
        .numExportedBuffers = (uint32_t)ExportID::NumExports,
        .numWorkers = (uint32_t)args.numWorkers,
    }, cfg, inits.data(), (madrona::CountT)TaskGraphID::NumTaskGraphs);

    const size_t W = (size_t)args.numWorlds;
    return oracle::runTrace(exec, args,
        { { (int)ExportID::Action, sizeof(Action) * kNumAgents } },
        { { (int)ExportID::Pairs, [=] { return W * sizeof(PairObs); } },
          { (int)ExportID::Zone, [=] { return W * sizeof(ZoneObs); } },
          { (int)ExportID::AgentPos, [=] { return W * kNumAgents * 12; } },
          { (int)ExportID::PickupEntity, [=] { return W * kNumPickups * 8; } },
          { (int)ExportID::PickupPos, [=] { return W * kNumPickups * 12; } },
          { (int)ExportID::PropEntity, [=] { return W * kNumProps * 8; } } });
}
