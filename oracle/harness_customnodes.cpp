// TEST INFRASTRUCTURE ONLY: sims/customnodes on the reference CPU backend, where its
// custom nodes are the reference's per-world addNodeFn form.  Built by oracle/customnodes.mk.
#include <madrona/mw_cpu.hpp>
#include "../sims/customnodes/sim.hpp"
#include "harness.hpp"

using namespace customnodes;

int main(int argc, char **argv)
{
    oracle::Args args = oracle::parseArgs(argc, argv);
    Config cfg {};
    std::vector<WorldInit> inits(args.numWorlds);
    for (int64_t i = 0; i < args.numWorlds; i++) {
        inits[i].seed = (uint32_t)(args.extra[0] + i);
        inits[i].empty = i % 7 == 3 ? 1u : 0u;
    }

    using Exec = madrona::TaskGraphExecutor<Engine, Sim, Config, WorldInit>;
    Exec exec({
        .numWorlds = (uint32_t)args.numWorlds,
        .numExportedBuffers = (uint32_t)ExportID::NumExports,
        .numWorkers = (uint32_t)args.numWorkers,
    }, cfg, inits.data(), (madrona::CountT)TaskGraphID::NumTaskGraphs);

    const size_t W = (size_t)args.numWorlds;
    // live tokens: Census::tokens of every world
    auto tokens = [&exec, W]() {
        const Census *c = (const Census *)exec.getExported((int)ExportID::Census);
        size_t n = 0;
        for (size_t i = 0; i < W; i++) n += c[i].tokens;
        return n;
    };
    return oracle::runTrace(exec, args, {},
        { { (int)ExportID::WorldSum, [=] { return W * sizeof(WorldSum); } },
          { (int)ExportID::CoopOut, [=] { return W * sizeof(CoopOut); } },
          { (int)ExportID::Census, [=] { return W * sizeof(Census); } },
          { (int)ExportID::TokenEntity, [=] { return tokens() * 8; } },
          { (int)ExportID::TokenVal, [=] { return tokens() * 4; } },
          { (int)ExportID::TokenOut, [=] { return tokens() * 4; } } });
}
