// TEST INFRASTRUCTURE ONLY: sims/crowd on the reference CPU backend (worlds of 20 to 1500
// bodies whose sizes change at every episode; --x0 seed, --x1 episode length, --x2 bodies
// per world for all worlds, 0: the fixture's sizes).  Built with -DCROWD_TWO_ARCHETYPES=1
// (crowd2), it also dumps the second archetype's columns.
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
    // rows of Body (second = false) or Body2 (second = true) in all worlds
    auto bodies = [&exec, W](bool second) {
        const BodyCount *counts = (const BodyCount *)exec.getExported((int)ExportID::BodyCount);
        size_t n = 0;
        for (size_t i = 0; i < W; i++) {
            int32_t body2 = 0;
#ifdef CROWD_TWO_ARCHETYPES
            body2 = counts[i].second;
#endif
            n += (size_t)(second ? body2 : counts[i].count - body2);
        }
        return n;
    };
    return oracle::runTrace(exec, args, {},
        { { (int)ExportID::BodyPos, [=] { return bodies(false) * 12; } },
          { (int)ExportID::BodyRot, [=] { return bodies(false) * 16; } },
          { (int)ExportID::BodyVel, [=] { return bodies(false) * 24; } },
          { (int)ExportID::BodyEntity, [=] { return bodies(false) * 8; } },
          { (int)ExportID::BodyCount, [=] { return W * sizeof(BodyCount); } },
#ifdef CROWD_TWO_ARCHETYPES
          { (int)ExportID::Body2Pos, [=] { return bodies(true) * 12; } },
          { (int)ExportID::Body2Rot, [=] { return bodies(true) * 16; } },
          { (int)ExportID::Body2Vel, [=] { return bodies(true) * 24; } },
          { (int)ExportID::Body2Entity, [=] { return bodies(true) * 8; } },
#endif
        });
}
