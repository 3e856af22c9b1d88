// TEST INFRASTRUCTURE ONLY: sims/crowd on the reference CPU backend (worlds of 20 to 1500
// bodies whose sizes change at every episode; --x0 seed, --x1 episode length, --x2 bodies
// per world for all worlds, 0: the fixture's sizes).
#include <madrona/mw_cpu.hpp>
#include "../sims/crowd/sim.hpp"
#include "harness.hpp"

using namespace crowd;

int main(int argc, char **argv)
{
    oracle::Args args = oracle::parseArgs(argc, argv);
    Config cfg {};
    cfg.objMgr = (madrona::phys::ObjectManager *)oracle::loadObjectsBlob(oracle::objectsPathArg(argc, argv));
    cfg.episodeLen = (uint32_t)args.extra[1];
    cfg.uniformBodies = (uint32_t)args.extra[2];
    cfg.layout = (uint32_t)Layout::Spread;
    std::vector<WorldInit> inits(args.numWorlds);
    for (int64_t i = 0; i < args.numWorlds; i++) inits[i].seed = (uint32_t)(args.extra[0] + i);

    using Exec = madrona::TaskGraphExecutor<Engine, Sim, Config, WorldInit>;
    Exec exec({
        .numWorlds = (uint32_t)args.numWorlds,
        .numExportedBuffers = (uint32_t)ExportID::NumExports,
        .numWorkers = (uint32_t)args.numWorkers,
    }, cfg, inits.data(), (madrona::CountT)TaskGraphID::NumTaskGraphs);

    const size_t W = (size_t)args.numWorlds;
    auto bodies = [&exec, W]() {
        const int32_t *counts = (const int32_t *)exec.getExported((int)ExportID::BodyCount);
        size_t n = 0;
        for (size_t i = 0; i < W; i++) n += (size_t)counts[i];
        return n;
    };
    return oracle::runTrace(exec, args, {},
        { { (int)ExportID::BodyPos, [=] { return bodies() * 12; } },
          { (int)ExportID::BodyRot, [=] { return bodies() * 16; } },
          { (int)ExportID::BodyVel, [=] { return bodies() * 24; } },
          { (int)ExportID::BodyEntity, [=] { return bodies() * 8; } },
          { (int)ExportID::BodyCount, [=] { return W * 4; } } });
}
