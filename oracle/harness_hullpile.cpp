// TEST INFRASTRUCTURE ONLY: sims/hullpile on the reference CPU backend (hulls at the
// engine's staging caps, compound bodies, spheres inside hulls, through the reference's
// own narrowphase + XPBD).  Always the pile layout.
#include <madrona/mw_cpu.hpp>
#include "../sims/hullpile/sim.hpp"
#include "harness.hpp"

using namespace hullpile;

int main(int argc, char **argv)
{
    oracle::Args args = oracle::parseArgs(argc, argv);
    Config cfg { (madrona::phys::ObjectManager *)oracle::loadObjectsBlob(oracle::objectsPathArg(argc, argv)),
                 (uint32_t)Layout::Pile, 0 };
    std::vector<WorldInit> inits(args.numWorlds);
    for (int64_t i = 0; i < args.numWorlds; i++) inits[i].seed = (uint32_t)(args.extra[0] + i);

    using Exec = madrona::TaskGraphExecutor<Engine, Sim, Config, WorldInit>;
    Exec exec({
        .numWorlds = (uint32_t)args.numWorlds,
        .numExportedBuffers = (uint32_t)ExportID::NumExports,
        .numWorkers = (uint32_t)args.numWorkers,
    }, cfg, inits.data(), (madrona::CountT)TaskGraphID::NumTaskGraphs);

    const size_t bodies = (size_t)args.numWorlds * kMaxBodies;
    return oracle::runTrace(exec, args, {},
        { { (int)ExportID::BodyPos, [=] { return bodies * 12; } },
          { (int)ExportID::BodyRot, [=] { return bodies * 16; } },
          { (int)ExportID::BodyVel, [=] { return bodies * 24; } },
          { (int)ExportID::BodyEntity, [=] { return bodies * 8; } },
          { (int)ExportID::BodyScale, [=] { return bodies * 12; } },
          { (int)ExportID::BodyObject, [=] { return bodies * 4; } } });
}
