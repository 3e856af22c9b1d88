// TEST INFRASTRUCTURE ONLY: sims/buttons on the reference CPU backend (XPBD step,
// then the reference's findEntitiesWithinAABB / checkEntityAABBOverlap on the
// refitted tree).  Built by oracle/overlap.mk.
#include <madrona/mw_cpu.hpp>
#include "../sims/buttons/sim.hpp"
#include "harness.hpp"

using namespace buttons;

int main(int argc, char **argv)
{
    oracle::Args args = oracle::parseArgs(argc, argv);
    Config cfg { (madrona::phys::ObjectManager *)oracle::loadObjectsBlob(oracle::objectsPathArg(argc, argv)),
                 (uint32_t)(args.extra[0] ? args.extra[0] : 100), 0 };
    std::vector<WorldInit> inits(args.numWorlds);
    for (int64_t i = 0; i < args.numWorlds; i++) inits[i].seed = (uint32_t)(args.extra[1] + i);

    using Exec = madrona::TaskGraphExecutor<Engine, Sim, Config, WorldInit>;
    Exec exec({
        .numWorlds = (uint32_t)args.numWorlds,
        .numExportedBuffers = (uint32_t)ExportID::NumExports,
        .numWorkers = (uint32_t)args.numWorkers,
    }, cfg, inits.data(), (madrona::CountT)TaskGraphID::NumTaskGraphs);

    const size_t W = (size_t)args.numWorlds;
    const size_t bodies = W * kNumPhysicsEntities;   // compacted at the end of every step
    return oracle::runTrace(exec, args,
        { { (int)ExportID::Reset, 4 }, { (int)ExportID::Action, sizeof(Action) * kNumAgents } },
        { { (int)ExportID::ButtonState, [=] { return W * kNumButtons * sizeof(ButtonState); } },
          { (int)ExportID::DoorPos, [=] { return W * kNumDoors * 12; } },
          { (int)ExportID::AgentPos, [=] { return W * kNumAgents * 12; } },
          { (int)ExportID::Goal, [=] { return W * kNumAgents * 4; } },
          { (int)ExportID::BodyPos, [=] { return bodies * 12; } },
          { (int)ExportID::BodyEntity, [=] { return bodies * 8; } } });
}
