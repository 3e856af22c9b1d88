// TEST INFRASTRUCTURE ONLY: sims/rays on the reference CPU backend (--x0 seed, --x1 episode
// length, --x2 bodies per world for all worlds, 0: the fixture's sizes, --x3 the largest of
// those sizes, 0: the fixture's default).  Dumps every ray
// row's inputs and its traceRay hit, the body counts and the bodies' positions and entities.
#include <madrona/mw_cpu.hpp>
#include "../sims/rays/sim.hpp"
#include "harness.hpp"

using namespace rays;

int main(int argc, char **argv)
{
    oracle::Args args = oracle::parseArgs(argc, argv);
    Config cfg {};
    cfg.objMgr = (madrona::phys::ObjectManager *)oracle::loadObjectsBlob(oracle::objectsPathArg(argc, argv));
    cfg.episodeLen = (uint32_t)args.extra[1];
    cfg.uniformBodies = (uint32_t)args.extra[2];
    cfg.variedBodies = (uint32_t)args.extra[3];
    std::vector<WorldInit> inits(args.numWorlds);
    for (int64_t i = 0; i < args.numWorlds; i++) inits[i].seed = (uint32_t)(args.extra[0] + i);

    using Exec = madrona::TaskGraphExecutor<Engine, Sim, Config, WorldInit>;
    Exec exec({
        .numWorlds = (uint32_t)args.numWorlds,
        .numExportedBuffers = (uint32_t)ExportID::NumExports,
        .numWorkers = (uint32_t)args.numWorkers,
    }, cfg, inits.data(), (madrona::CountT)TaskGraphID::NumTaskGraphs);

    const size_t W = (size_t)args.numWorlds;
    const size_t R = W * (size_t)kRaysPerWorld;
    auto bodies = [&exec, W] {
        const BodyCount *counts = (const BodyCount *)exec.getExported((int)ExportID::BodyCount);
        size_t n = 0;
        for (size_t i = 0; i < W; i++) n += (size_t)counts[i].count;
        return n;
    };
    return oracle::runTrace(exec, args, {},
        { { (int)ExportID::RayOrigin, [=] { return R * 12; } },
          { (int)ExportID::RayDir, [=] { return R * 12; } },
          { (int)ExportID::RayMaxT, [=] { return R * 4; } },
          { (int)ExportID::HitEntity, [=] { return R * 8; } },
          { (int)ExportID::HitT, [=] { return R * 4; } },
          { (int)ExportID::HitNormal, [=] { return R * 12; } },
          { (int)ExportID::BodyCount, [=] { return W * sizeof(BodyCount); } },
          { (int)ExportID::BodyPos, [=] { return bodies() * 12; } },
          { (int)ExportID::BodyEntity, [=] { return bodies() * 8; } } });
}
