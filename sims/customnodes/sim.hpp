// Fixture simulator for custom task-graph nodes (TaskGraphBuilder::addNodeFn,
// addOneOffNode, addDynamicCountNode, node data).  ECS only, integer state.
//
// The same sources build against the reference CPU backend, where a custom node is
// fn(NodeT *, Context &, TaskGraph &) called once per world, and against the GPU
// engine, where it is fn(NodeT *, int32_t invocation) over all worlds.  Both forms
// compute the same exported columns bit for bit:
//   * SpawnNode (fixed count = worlds, 1 thread each): per-world token churn through
//     TaskGraph::makeContext -- values change, tokens die and are born, some worlds stay
//     empty, and every 9th step leaves no token anywhere;
//   * WarpSumNode (fixed count = worlds, 32 threads each): a warp-per-world reduction;
//   * TokenRowsNode (addDynamicCountNode): one invocation per live Token row, through a
//     QueryRef taken in the constructor;
//   * SetCountNode (addOneOffNode<.., 1>) sets CoopNode's numDynamicInvocations through
//     getNodeData; CoopNode (256 threads per invocation, __shared__ + __syncthreads)
//     zeroes its own count while it runs;
//   * CensusNode in a second task graph.
// The three branches after the compaction run on parallel graph branches.
//
// Build variants (GPU only):
//   CUSTOMNODES_PROBE=1: a node with a fixed count N and T threads per invocation (both
//     from Config) records every run it gets into kProbeSlots fixed rows;
//   CUSTOMNODES_BENCH=1: the TokenRowsNode work again as a ParallelForNode.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>
#include <madrona/rand.hpp>

namespace customnodes {

using madrona::Entity;
using madrona::CountT;

constexpr int32_t kMaxTokens = 20;
constexpr int32_t kMaxCoop = 6;
constexpr int32_t kProbeSlots = 4096;

enum class ExportID : uint32_t {
    WorldSum,
    CoopOut,
    Census,
    TokenEntity,
    TokenVal,
    TokenOut,
    ProbeRec,
    ProbeInfo,
    NumExports,
};

enum class TaskGraphID : uint32_t {
    Step,
    Census,
    NumTaskGraphs,
};

struct TokenVal { uint32_t v; };
struct TokenOut { uint32_t h; };

// per world: live tokens, wrapping sum of their values, XOR of their entity IDs, largest value
struct WorldSum { uint32_t count; uint32_t sum; uint32_t xorIDs; uint32_t maxVal; };
// per world: this step's block count k and the k block-cooperative sums
struct CoopOut { uint32_t k; uint32_t v[kMaxCoop]; };
struct Census { uint32_t calls; uint32_t tokens; uint32_t made; uint32_t pad; };

// probe rows: lane executions, sums of invocation and lane indices, lanes seen (bit per lane)
struct ProbeRec {
    uint32_t hits;
    uint32_t pad;
    unsigned long long invSum;
    unsigned long long laneSum;
    uint32_t lanes[8];
};
// largest invocation index that ran, plus one
struct ProbeInfo { uint32_t maxInvPlus1; uint32_t pad; };

struct Token : public madrona::Archetype<TokenVal, TokenOut> {};
struct ProbeSlot : public madrona::Archetype<ProbeRec> {};

struct Config {
    uint32_t probeCount;       // probe build: N (0: dynamic with a count of 0)
    uint32_t probeThreads;     // probe build: T
    uint32_t probeDynamic;     // probe build: N is set by a one-off node; invocation 0 zeroes it
    uint32_t extraNodeDatas;   // probe build: node datas constructed beyond the graph's own
};

struct WorldInit {
    uint32_t seed;
    uint32_t empty;            // the world never has tokens
};

class Engine;

struct Sim : public madrona::WorldBase {
    static void registerTypes(madrona::ECSRegistry &registry, const Config &cfg);
    static void setupTasks(madrona::TaskGraphManager &mgr, const Config &cfg);

    Sim(Engine &ctx, const Config &cfg, const WorldInit &init);

    madrona::RNG rng;
    Entity tokens[kMaxTokens];
    int32_t numTokens;
    uint32_t empty;
    uint32_t salt;
    uint32_t curStep;
    uint32_t totalMade;
    uint32_t coopK;            // CPU backend: this step's k, from SetCountNode
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
