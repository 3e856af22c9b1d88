// GPU-only fixture that drives the archetype sort / compaction kernels through
// their edges: row counts around the 2048-row tile, world counts where the
// number of world-sort passes changes, every column width the rearrange kernel
// moves in its own unit type, exported and non-exported columns, empty worlds
// and steps that delete whole worlds or the whole table.
//
// Every byte of every row is a pure function of (world, uid, component, byte
// index) and every key a pure function of (world seed, uid, step), so
// tests/test_sort_sweep.py predicts the whole table with a numpy model of the
// churn and oracle/restate.py's sort semantics.  After the sorts a row system
// recomputes each row's bytes and checks the row's entity slot, writing any
// mismatch into Check; a per-world system hashes the world's rows in query
// order into Summary, which pins worldOffsets / worldCounts.
#pragma once

#include <madrona/taskgraph_builder.hpp>
#include <madrona/custom_context.hpp>

namespace sortsweep {

using madrona::Entity;

enum class ExportID : uint32_t {
    Entity, Uid, Key4, Check, P2, P3, P12, P24, P48, Summary, NumExports,
};
enum class TaskGraphID : uint32_t { Step, NumTaskGraphs };

// graph shapes (Config::shape)
enum Shape : uint32_t {
    ShapeSort = 0,          // rekey -> custom sort
    ShapeChurn = 1,         // churn -> compact
    ShapeRekeyChurnSort = 2,// rekey -> churn -> custom sort (sees destroyed rows) -> compact
};
// key distributions (Config::keyMode)
enum KeyMode : uint32_t {
    KeyUniform = 0,         // 32 random bits, one key in 16 forced to 0xFFFFFFFF
    KeyConstant = 1,        // every key equal
    KeyAllOnes = 2,         // every key 0xFFFFFFFF
    KeyByte3 = 3,           // only bits 24..31 vary
};

struct Uid { uint32_t v; };
struct Key4 { uint32_t v; };
struct Key8 { uint32_t v; uint32_t hi; };   // key in the first 4 bytes
struct P1 { uint8_t b[1]; };
struct P2 { uint8_t b[2]; };
struct P3 { uint8_t b[3]; };
struct P5 { uint8_t b[5]; };
struct P8 { uint8_t b[8]; };
struct P12 { uint8_t b[12]; };
struct P20 { uint8_t b[20]; };
struct P24 { uint8_t b[24]; };
struct P32 { uint8_t b[32]; };
struct P48 { uint8_t b[48]; };
struct P6 { uint8_t b[6]; };                // payload 10: a 2-byte unit on the flip path
struct Check { uint32_t mismatch; };        // bit 0 entity slot, 1 Key4, 2 Key8, 3 + i payload i
struct StepCounter { uint32_t t; };
struct Summary { uint32_t count; uint32_t hash; };

struct Item : public madrona::Archetype<
    Uid, Key4, Key8, P1, P2, P3, P5, P8, P12, P20, P24, P32, P48, P6, Check
> {};

struct Config {
    uint32_t shape;
    uint32_t keyMode;
    uint32_t sortOnKey8;        // custom sort on Key8 instead of Key4
    uint32_t destroyThreshold;  // a row dies at step t when hashOf(seed, uid, t) < this
};

struct WorldInit {
    uint32_t seed;
    uint32_t initCount;         // items made by the constructor
    uint32_t createsPerStep;    // items made by every step's churn
    uint32_t killStep;          // at this step the world destroys every item and makes none (0: never)
};

// ---- pure functions shared with the test's numpy model ----
inline uint32_t mix32(uint32_t h)
{
    h ^= h >> 16;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    h *= 0xC2B2AE35u;
    h ^= h >> 16;
    return h;
}

inline uint32_t hashOf(uint32_t seed, uint32_t uid, uint32_t t)
{
    return mix32(seed ^ mix32(uid * 0x9E3779B1u + t * 0x7F4A7C15u + 1u));
}

inline uint32_t keyOf(uint32_t seed, uint32_t uid, uint32_t t, uint32_t mode)
{
    const uint32_t r = hashOf(seed ^ 0x5BD1E995u, uid, t);
    switch (mode) {
    case KeyConstant: return 0x2A2A2A2Au;
    case KeyAllOnes: return 0xFFFFFFFFu;
    case KeyByte3: return r & 0xFF000000u;
    default: return (r & 0xFu) == 0 ? 0xFFFFFFFFu : r;
    }
}

inline uint32_t key8Hi(uint32_t key, uint32_t uid)
{
    return ~key ^ (uid * 0x01000193u);
}

// byte i of payload component c of row (world, uid)
inline uint8_t payloadByte(uint32_t world, uint32_t uid, uint32_t c, uint32_t i)
{
    const uint32_t row = mix32(uid * 0x9E3779B1u + world * 0x85EBCA77u + 1u);
    const uint32_t h = mix32(row + c * 0x27D4EB2Fu);
    return (uint8_t)((h >> (8u * (i & 3u))) + 0x3Bu * (i >> 2));
}

// order-sensitive hash of the uids a world's query visits, the i-th one adding mix32(uid + i * golden)
inline uint32_t summaryTerm(uint32_t uid, uint32_t i)
{
    return mix32(uid + i * 0x9E3779B9u);
}

class Engine;

struct Sim : public madrona::WorldBase {
    static void registerTypes(madrona::ECSRegistry &registry, const Config &cfg);
    static void setupTasks(madrona::TaskGraphManager &mgr, const Config &cfg);
    Sim(Engine &ctx, const Config &cfg, const WorldInit &init);

    uint32_t seed;
    uint32_t nextUid;
    uint32_t createsPerStep;
    uint32_t killStep;
    uint32_t shape;
    uint32_t keyMode;
    uint32_t destroyThreshold;
};

class Engine : public madrona::CustomContext<Engine, Sim> {
public:
    using CustomContext::CustomContext;
};

}
