// Compiler glue.  MADRONA_GPU_MODE is defined on the NVRTC command line
// (same macro the reference defines for its device build: src/mw/CMakeLists.txt:38-47).
#pragma once
#if defined(__CUDACC__)
#define MB2_HD __host__ __device__
#else
#define MB2_HD
#endif
#define MADRONA_ALWAYS_INLINE __attribute__((always_inline))
#define MADRONA_NO_INLINE __attribute__((noinline))
#define MADRONA_UNROLL _Pragma("unroll")
#define MADRONA_UNREACHABLE() __builtin_unreachable()
#ifdef MADRONA_GPU_MODE
#define MADRONA_GPU_COND(...) __VA_ARGS__
#else
#define MADRONA_GPU_COND(...)
#endif
#define MADRONA_MW_COND(...) __VA_ARGS__
#define MADRONA_CACHE_LINE 128
#define MADRONA_EXPORT
#define MADRONA_IMPORT
#if defined(__CUDA_ARCH__) || defined(__CUDACC_RTC__)
#define MB2_CLZ(v) __clz((int)(v))
#define MB2_CLZLL(v) __clzll((long long)(v))
#define MB2_POPC(v) __popc((unsigned)(v))
#else
#define MB2_CLZ(v) __builtin_clz(v)
#define MB2_CLZLL(v) __builtin_clzll(v)
#define MB2_POPC(v) __builtin_popcount(v)
#endif
