// Reference: include/madrona/memory.hpp:26-37, 164-168 and, for the GPU backend,
// src/mw/device/include/madrona/memory.hpp:17-43.
//
// On the device, rawAlloc / rawAllocAligned carve from the engine's persistent arena
// (EngineState::persistArena, sized by MADRONA_B200_PERSIST_BYTES), the arena that
// phys::init carves per-world broadphase storage from.  The reference puts them on a
// device malloc heap instead (MADRONA_MWGPU_DEVICE_HEAP_SIZE, not honoured here).
//   * World constructors run in two or more passes (a dry run first); the arena is
//     rewound to the same mark before each pass, so what a pass allocated is reclaimed
//     and only the last pass's allocations stay.
//   * Allocations from setupTasks or from step kernels are never returned: rawDealloc
//     is a no-op, and the arena only grows until the executor is destroyed.
//   * A full arena raises ErrPersistOverflow (reported as "persistent arena overflow
//     (raise MADRONA_B200_PERSIST_BYTES)") and returns nullptr.
// Host builds (the engine's host tools and probes) use malloc, as the reference does.
#pragma once
#include <cstddef>
#include <cstdint>
#include <madrona/macros.hpp>
#ifdef MADRONA_GPU_MODE
#include <madrona/state.hpp>
#else
#include <cstdlib>
#endif

namespace madrona {

#ifdef MADRONA_GPU_MODE
namespace mwGPU {
// Every persistent carve is a multiple of 128 bytes (phys::init rounds the same way), so
// each one starts 128-byte aligned in the 256-aligned arena.
inline void *persistAlloc(uint64_t num_bytes)
{
    mb2::EngineState &S = engine();
    num_bytes = (num_bytes + 127ull) & ~127ull;
    unsigned long long off = atomicAdd((unsigned long long *)&S.persistOffset,
                                       (unsigned long long)num_bytes);
    if (off + num_bytes > S.persistCapacity) {
        raiseError(mb2::ErrPersistOverflow);
        return nullptr;
    }
    return S.persistArena + off;
}

// Context-free bump allocation from the tmp arena (what Context::tmpAlloc does): rewound
// by ResetTmpAllocNode and before every world-construction pass.
inline void *tmpArenaAlloc(uint64_t num_bytes)
{
    mb2::EngineState &S = engine();
    num_bytes = (num_bytes + 255ull) & ~255ull;
    unsigned long long off = atomicAdd((unsigned long long *)&S.tmpOffset,
                                       (unsigned long long)num_bytes);
    if (off + num_bytes > S.tmpCapacity) {
        raiseError(mb2::ErrTmpOverflow);
        return nullptr;
    }
    return S.tmpArena + off;
}
}

inline void *rawAlloc(size_t num_bytes)
{
    return mwGPU::persistAlloc(num_bytes);
}

// alignment: a power of 2
inline void *rawAllocAligned(size_t num_bytes, size_t alignment)
{
    if (alignment <= 128) {
        return mwGPU::persistAlloc(num_bytes);
    }
    char *p = (char *)mwGPU::persistAlloc(num_bytes + alignment);
    if (p == nullptr) {
        return nullptr;
    }
    uintptr_t a = ((uintptr_t)p + alignment - 1) & ~(uintptr_t)(alignment - 1);
    return (void *)a;
}

inline void rawDealloc(void *) {}
inline void rawDeallocAligned(void *) {}
#else
inline void *rawAlloc(size_t num_bytes) { return malloc(num_bytes); }
inline void *rawAllocAligned(size_t num_bytes, size_t alignment)
{
    return aligned_alloc(alignment, (num_bytes + alignment - 1) / alignment * alignment);
}
inline void rawDealloc(void *ptr) { free(ptr); }
inline void rawDeallocAligned(void *ptr) { free(ptr); }
#endif

class DefaultAlloc {
public:
    inline void *alloc(size_t num_bytes) { return rawAlloc(num_bytes); }
    inline void dealloc(void *ptr) { rawDealloc(ptr); }
};

using InitAlloc = DefaultAlloc;
using TmpAlloc = DefaultAlloc;

}
