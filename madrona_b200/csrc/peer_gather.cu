// peer_gather.cu -- multi-GPU gather of exported columns by direct NVLink
// peer stores (SURVEY.md 8e: worlds shard across GPUs, the only exchange is the
// observation / reward / done gather into the world-major tensor every rank
// sees).  The reference is single-GPU (include/madrona/mw_gpu.hpp:122), so
// there is no counterpart to cite; the mechanism replaces "one NCCL
// all_gather per exported tensor per step":
//
//   * every rank owns a SYMMETRIC buffer  [2 parities][slot][world_size][bytes_slot]
//     in its own HBM, exported through cudaIpc so every peer maps it (or, for
//     ranks of one process on one GPU, handed over by connect_local);
//   * after its step graph, ONE kernel per rank reads the rank's exported
//     columns once (16-byte loads) and stores them into slice `rank` of every
//     peer's buffer (16-byte NVLink stores, 8- or 4-byte ones into a slice that
//     starts off a 16-byte boundary; peers interleaved per thread so all links
//     are busy), then publishes `arrived[rank] = step + 1` on every peer
//     behind a __threadfence_system();
//   * consumers wait on the flags (a 1-warp spin kernel), read the gathered
//     tensors of parity step & 1, and release the parity so the pushers of step
//     + 2 may overwrite it (flow control through `released[rank]` flags written
//     the same way).
// No host round trip, no rank barrier, no extra copy: the gather of step t
// overlaps the step graph of t + 1 on every rank.
#include "../../include/madrona_b200.h"
#include "engine.hpp"

#include <cstring>
#include <vector>

namespace mb2 {

constexpr int kMaxGatherSlots = 8;
constexpr int kMaxPeers = 16;

struct GatherFlags {
    // written by peer r (slot r), read by the owner
    unsigned long long arrived[kMaxPeers];    // steps pushed so far by r
    unsigned long long released[kMaxPeers];   // steps r has finished reading
};

struct GatherDevice {
    // this rank's view of every rank's symmetric buffer / flags (index = rank)
    char *peerData[kMaxPeers];
    GatherFlags *peerFlags[kMaxPeers];
    const char *src[kMaxGatherSlots];          // exported columns of this rank
    unsigned long long slotBytes[kMaxGatherSlots];
    unsigned long long slotOffset[kMaxGatherSlots];   // inside one parity, of [world_size][bytes]
    unsigned long long parityBytes;
    unsigned int numSlots;
    unsigned int worldSize;
    unsigned int rank;
    unsigned int blocksDone;
    unsigned long long pushStep;       // steps this rank has pushed
    unsigned long long waitStep;       // steps this rank has waited for
    unsigned long long releaseStep;    // steps this rank has released
};

struct PeerGather {
    Executor *ex = nullptr;
    GatherDevice host;
    GatherDevice *dev = nullptr;
    char *localData = nullptr;
    GatherFlags *localFlags = nullptr;
    std::vector<void *> opened;
    uint64_t hostPushes = 0;
};

__device__ __forceinline__ unsigned long long loadSys(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void storeSys(unsigned long long *p, unsigned long long v)
{
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}

// Stores vector i of a slice (its bytes 16 i .. 16 i + 15) as kWidth-byte stores.
template <int kWidth>
__device__ __forceinline__ void storeVector(char *slice, unsigned long long i, const uint4 &v)
{
    if constexpr (kWidth == 16) {
        reinterpret_cast<uint4 *>(slice)[i] = v;
    } else if constexpr (kWidth == 8) {
        uint2 *d = reinterpret_cast<uint2 *>(slice) + 2 * i;
        d[0] = make_uint2(v.x, v.y);
        d[1] = make_uint2(v.z, v.w);
    } else {
        unsigned int *d = reinterpret_cast<unsigned int *>(slice) + 4 * i;
        d[0] = v.x;
        d[1] = v.y;
        d[2] = v.z;
        d[3] = v.w;
    }
}

// The whole 16-byte vectors of one slot: 16-byte loads from the exported column, kWidth-byte
// stores into every peer's slice at dst_off.
template <int kWidth>
__device__ __forceinline__ void pushVectors(const GatherDevice &G, const uint4 *src, unsigned long long vecs,
                                            unsigned long long dst_off)
{
    const unsigned int P = G.worldSize;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < vecs;
         i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint4 v = src[i];
        // start at a different peer per thread group so the stores spread over all links.
        // Unrolling the narrow variants too would spill the slot's state to local memory.
#pragma unroll (kWidth == 16 ? 4 : 1)
        for (unsigned int k = 0; k < P; k++) {
            const unsigned int peer = (k + G.rank + 1u + (unsigned int)(i >> 5)) % P;
            storeVector<kWidth>(G.peerData[peer] + dst_off, i, v);
        }
    }
}

// Push step s = G.pushStep: wait until every peer released step s - 2 (the
// previous user of this parity), copy, publish.
__global__ void __launch_bounds__(256)
gatherPushKernel(GatherDevice *Gp)
{
    GatherDevice &G = *Gp;
    const unsigned long long step = G.pushStep;
    const unsigned int parity = (unsigned int)(step & 1ull);
    const unsigned int P = G.worldSize;

    if (step >= 2) {
        // flow control: peer r must have finished reading step - 2 out of ITS
        // buffer before this rank overwrites its slice there; r records that in
        // this rank's flags block
        if (threadIdx.x < P) {
            const GatherFlags *mine = G.peerFlags[G.rank];
            while (loadSys(&mine->released[threadIdx.x]) < step - 1) __nanosleep(64);
        }
        __syncthreads();
    }

    for (unsigned int s = 0; s < G.numSlots; s++) {
        const unsigned long long bytes = G.slotBytes[s];
        const unsigned long long vecs = bytes >> 4;
        const uint4 *src = reinterpret_cast<const uint4 *>(G.src[s]);
        const unsigned long long dst_off = (unsigned long long)parity * G.parityBytes + G.slotOffset[s] +
            (unsigned long long)G.rank * bytes;
        // parityBytes and slotOffset are multiples of 256, so the slice of rank r starts at
        // r * bytes modulo 16: only 4-byte aligned when bytes is not a multiple of 16.  The
        // offset is the same on every peer, so one store width serves the whole slot.
        if ((dst_off & 15ull) == 0) {
            pushVectors<16>(G, src, vecs, dst_off);
        } else if ((dst_off & 7ull) == 0) {
            pushVectors<8>(G, src, vecs, dst_off);
        } else {
            pushVectors<4>(G, src, vecs, dst_off);
        }
        // tail (columns are 4-byte multiples)
        const unsigned long long tail_words = (bytes & 15ull) >> 2;
        if (blockIdx.x == 0 && threadIdx.x < tail_words) {
            const unsigned int w = ((const unsigned int *)G.src[s])[(vecs << 2) + threadIdx.x];
            for (unsigned int peer = 0; peer < P; peer++) {
                ((unsigned int *)(G.peerData[peer] + dst_off))[(vecs << 2) + threadIdx.x] = w;
            }
        }
    }

    // last block out publishes the step on every peer
    __shared__ bool is_last;
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int done = atomicAdd(&G.blocksDone, 1u);
        is_last = done == gridDim.x - 1;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence_system();
    if (threadIdx.x < P) storeSys(&G.peerFlags[threadIdx.x]->arrived[G.rank], step + 1);
    if (threadIdx.x == 0) {
        G.blocksDone = 0;
        G.pushStep = step + 1;
    }
}

// Wait until the slices of step s = G.waitStep of ALL ranks sit in this rank's buffer.
__global__ void gatherWaitKernel(GatherDevice *Gp)
{
    GatherDevice &G = *Gp;
    const unsigned long long step = G.waitStep;
    if (threadIdx.x < G.worldSize) {
        const GatherFlags *mine = G.peerFlags[G.rank];
        while (loadSys(&mine->arrived[threadIdx.x]) < step + 1) __nanosleep(64);
    }
    __syncthreads();
    if (threadIdx.x == 0) G.waitStep = step + 1;
}

// This rank is done reading step s = G.releaseStep: tell every pusher.
__global__ void gatherReleaseKernel(GatherDevice *Gp)
{
    GatherDevice &G = *Gp;
    const unsigned long long step = G.releaseStep;
    __threadfence_system();
    if (threadIdx.x < G.worldSize) storeSys(&G.peerFlags[threadIdx.x]->released[G.rank], step + 1);
    if (threadIdx.x == 0) G.releaseStep = step + 1;
}

}

using namespace mb2;

extern "C" {

mb2_peer_gather *mb2_peer_gather_create(mb2_executor *exec, const int64_t *slots, uint32_t num_slots,
                                        const uint64_t *bytes_per_slot, uint32_t world_size, uint32_t rank)
{
    Executor *ex = (Executor *)exec;
    const std::string fn = "mb2_peer_gather_create: ";
    std::string err;
    if (!ex) {
        err = "null executor";
    } else if (num_slots == 0 || num_slots > (uint32_t)kMaxGatherSlots) {
        err = "num_slots must be 1 to " + std::to_string(kMaxGatherSlots) + ", got " + std::to_string(num_slots);
    } else if (world_size == 0 || world_size > (uint32_t)kMaxPeers) {
        err = "world_size must be 1 to " + std::to_string(kMaxPeers) + ", got " + std::to_string(world_size);
    } else if (rank >= world_size) {
        err = "rank " + std::to_string(rank) + " is not below world_size " + std::to_string(world_size);
    } else if (!slots || !bytes_per_slot) {
        err = "null slots or bytes_per_slot";
    }
    for (uint32_t s = 0; err.empty() && s < num_slots; s++) {
        if (!mb2_get_exported(exec, slots[s])) {
            err = "export slot " + std::to_string(slots[s]) + " (entry " + std::to_string(s) + ") is not in use";
        } else if (bytes_per_slot[s] & 3ull) {
            // any multiple of 4 works: the push kernel narrows its stores to the slice's alignment
            err = "entry " + std::to_string(s) + ": " + std::to_string(bytes_per_slot[s]) +
                  " bytes per rank is not a multiple of 4";
        }
    }
    if (!err.empty()) {
        setError(fn + err);
        return nullptr;
    }
    cudaSetDevice(ex->gpu);
    PeerGather *g = new PeerGather();
    g->ex = ex;
    GatherDevice &G = g->host;
    memset(&G, 0, sizeof(G));
    G.numSlots = num_slots;
    G.worldSize = world_size;
    G.rank = rank;
    unsigned long long off = 0;
    for (uint32_t s = 0; s < num_slots; s++) {
        G.src[s] = (const char *)mb2_get_exported(exec, slots[s]);
        G.slotBytes[s] = bytes_per_slot[s];
        G.slotOffset[s] = off;
        off += ((bytes_per_slot[s] * world_size + 255ull) & ~255ull);
    }
    G.parityBytes = off;
    if (cudaMalloc((void **)&g->localData, 2 * off) != cudaSuccess ||
        cudaMalloc((void **)&g->localFlags, sizeof(GatherFlags)) != cudaSuccess ||
        cudaMalloc((void **)&g->dev, sizeof(GatherDevice)) != cudaSuccess) {
        setError("mb2_peer_gather_create: allocation failed");
        delete g;
        return nullptr;
    }
    cudaMemset(g->localData, 0, 2 * off);
    cudaMemset(g->localFlags, 0, sizeof(GatherFlags));
    cudaDeviceSynchronize();
    return (mb2_peer_gather *)g;
}

int mb2_peer_gather_local_handle(mb2_peer_gather *gather, void *handle_out)
{
    PeerGather *g = (PeerGather *)gather;
    cudaIpcMemHandle_t h[2];
    if (cudaIpcGetMemHandle(&h[0], g->localData) != cudaSuccess ||
        cudaIpcGetMemHandle(&h[1], g->localFlags) != cudaSuccess) {
        setError(std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(cudaGetLastError()));
        return 1;
    }
    memcpy(handle_out, h, sizeof(h));
    return 0;
}

int mb2_peer_gather_connect(mb2_peer_gather *gather, const void *all_handles)
{
    PeerGather *g = (PeerGather *)gather;
    GatherDevice &G = g->host;
    cudaSetDevice(g->ex->gpu);
    const cudaIpcMemHandle_t *h = (const cudaIpcMemHandle_t *)all_handles;
    for (uint32_t r = 0; r < G.worldSize; r++) {
        if (r == G.rank) {
            G.peerData[r] = g->localData;
            G.peerFlags[r] = g->localFlags;
            continue;
        }
        void *data = nullptr, *flags = nullptr;
        if (cudaIpcOpenMemHandle(&data, h[2 * r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess ||
            cudaIpcOpenMemHandle(&flags, h[2 * r + 1], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
            setError(std::string("cudaIpcOpenMemHandle (rank ") + std::to_string(r) + "): " +
                     cudaGetErrorString(cudaGetLastError()));
            return 1;
        }
        g->opened.push_back(data);
        g->opened.push_back(flags);
        G.peerData[r] = (char *)data;
        G.peerFlags[r] = (GatherFlags *)flags;
    }
    if (cudaMemcpy(g->dev, &G, sizeof(G), cudaMemcpyHostToDevice) != cudaSuccess) {
        setError("mb2_peer_gather_connect: upload failed");
        return 1;
    }
    return 0;
}

int mb2_peer_gather_connect_local(mb2_peer_gather *const *gathers, uint32_t n)
{
    // everything is checked before any gather changes, so a refused call leaves them as they were
    std::string err;
    if (!gathers || n == 0) err = "no gathers";
    for (uint32_t r = 0; err.empty() && r < n; r++) {
        if (!gathers[r]) err = "gathers[" + std::to_string(r) + "] is null";
    }
    std::vector<int> seen(n, -1);
    for (uint32_t r = 0; err.empty() && r < n; r++) {
        const PeerGather *g = (const PeerGather *)gathers[r];
        const PeerGather *g0 = (const PeerGather *)gathers[0];
        const std::string at = "gathers[" + std::to_string(r) + "] ";
        if (g->host.worldSize != n) {
            err = at + "has world_size " + std::to_string(g->host.worldSize) + ", but " + std::to_string(n) +
                  " gathers were given";
        } else if (seen[g->host.rank] >= 0) {
            err = "rank " + std::to_string(g->host.rank) + " appears twice (gathers[" +
                  std::to_string(seen[g->host.rank]) + "] and gathers[" + std::to_string(r) + "])";
        } else if (g->host.rank != r) {
            err = at + "is rank " + std::to_string(g->host.rank) + "; gathers[r] must be rank r's gather";
        } else if (g->host.numSlots != g0->host.numSlots) {
            err = at + "has " + std::to_string(g->host.numSlots) + " slots, gathers[0] " +
                  std::to_string(g0->host.numSlots);
        } else if (g->ex->gpu != g0->ex->gpu) {
            err = at + "is on GPU " + std::to_string(g->ex->gpu) + ", gathers[0] on GPU " +
                  std::to_string(g0->ex->gpu);
        }
        for (uint32_t s = 0; err.empty() && s < g->host.numSlots; s++) {
            if (g->host.slotBytes[s] != g0->host.slotBytes[s]) {
                err = at + "slot " + std::to_string(s) + " has " + std::to_string(g->host.slotBytes[s]) +
                      " bytes per rank, gathers[0] " + std::to_string(g0->host.slotBytes[s]);
            }
        }
        if (err.empty()) seen[g->host.rank] = (int)r;
    }
    if (!err.empty()) {
        setError("mb2_peer_gather_connect_local: " + err);
        return 1;
    }
    for (uint32_t r = 0; r < n; r++) {
        PeerGather *g = (PeerGather *)gathers[r];
        for (uint32_t p = 0; p < n; p++) {
            g->host.peerData[p] = ((PeerGather *)gathers[p])->localData;
            g->host.peerFlags[p] = ((PeerGather *)gathers[p])->localFlags;
        }
        cudaSetDevice(g->ex->gpu);
        if (cudaMemcpy(g->dev, &g->host, sizeof(g->host), cudaMemcpyHostToDevice) != cudaSuccess) {
            setError("mb2_peer_gather_connect_local: upload failed");
            return 1;
        }
    }
    return 0;
}

int mb2_peer_gather_push_async(mb2_peer_gather *gather, void *cuda_stream)
{
    PeerGather *g = (PeerGather *)gather;
    unsigned long long max_bytes = 0;
    for (uint32_t s = 0; s < g->host.numSlots; s++) max_bytes = std::max<unsigned long long>(max_bytes, g->host.slotBytes[s]);
    unsigned blocks = (unsigned)std::max<unsigned long long>(1, std::min<unsigned long long>((max_bytes / 16 + 255) / 256, 32));
    gatherPushKernel<<<blocks, 256, 0, (cudaStream_t)cuda_stream>>>(g->dev);
    g->hostPushes++;
    return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

int mb2_peer_gather_wait_async(mb2_peer_gather *gather, void *cuda_stream)
{
    PeerGather *g = (PeerGather *)gather;
    gatherWaitKernel<<<1, 32, 0, (cudaStream_t)cuda_stream>>>(g->dev);
    return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

int mb2_peer_gather_release_async(mb2_peer_gather *gather, void *cuda_stream)
{
    PeerGather *g = (PeerGather *)gather;
    gatherReleaseKernel<<<1, 32, 0, (cudaStream_t)cuda_stream>>>(g->dev);
    return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

void *mb2_peer_gather_buffer(mb2_peer_gather *gather, uint32_t parity, uint32_t slot_index)
{
    PeerGather *g = (PeerGather *)gather;
    if (!g || slot_index >= g->host.numSlots || parity > 1) return nullptr;
    return g->localData + (size_t)parity * g->host.parityBytes + g->host.slotOffset[slot_index];
}

void mb2_peer_gather_destroy(mb2_peer_gather *gather)
{
    PeerGather *g = (PeerGather *)gather;
    if (!g) return;
    cudaSetDevice(g->ex->gpu);
    cudaDeviceSynchronize();
    for (void *p : g->opened) cudaIpcCloseMemHandle(p);
    cudaFree(g->localData);
    cudaFree(g->localFlags);
    cudaFree(g->dev);
    delete g;
}

}
