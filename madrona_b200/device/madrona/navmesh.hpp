// Reference: include/madrona/navmesh.{hpp,inl}, src/common/navmesh.cpp.
//
// Navigation meshes: polygons fanned into triangles, an alias table for area-weighted
// point sampling, triangle adjacency, breadth-first search and Dijkstra over triangles.
// Same layout and bit-identical results as the reference CPU backend:
//   * the mesh arrays are read through the read-only data path (__ldg) on the device;
//   * the searches run entirely out of caller scratch (BFSState / DijkstrasState), so
//     one thread per agent can search inside any node; the callbacks are inlined;
//   * the heap keeps the reference's tie rules, which decide the visit order among
//     equal costs: sift-up stops at a parent of equal cost, sift-down takes the right
//     child only when strictly cheaper and stops only when strictly below the child.
//
// initFromPolygons on the device (world constructors, setupTasks, step kernels) puts the
// four arrays in the persistent arena (rawAlloc) and its temporaries -- weights, the two
// alias stacks and the edge map, about 60 bytes per triangle -- in the tmp arena.  A
// polygon of fewer than 3 vertices raises ErrNavmeshPolygon and nothing is built; so does
// a full arena (ErrPersistOverflow / ErrTmpOverflow).  A mesh that was not built has
// numTris == 0 and null arrays.
#pragma once
#include <cfloat>
#include <cstddef>
#include <cstdint>
#include <madrona/math.hpp>
#include <madrona/rand.hpp>
#include <madrona/utils.hpp>
#include <madrona/memory.hpp>

#if defined(__CUDACC__) || defined(__CUDACC_RTC__)
#define MB2_NAVMESH_UNROLL _Pragma("unroll")
#else
#define MB2_NAVMESH_UNROLL
#endif

namespace madrona {

namespace navmeshRO {
MB2_HD inline uint32_t ld(const uint32_t *__restrict__ p)
{
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}
MB2_HD inline float ld(const float *__restrict__ p)
{
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}
MB2_HD inline math::Vector3 ldVec3(const math::Vector3 *__restrict__ p)
{
    const float *f = (const float *)p;
    return math::Vector3 { ld(f), ld(f + 1), ld(f + 2) };
}
}

struct Navmesh {
    struct PathFindQueue {
        float *costs;
        uint32_t *heap;
        uint32_t *heapIndex;
        CountT heapSize;

        MB2_HD inline void add(uint32_t poly, float cost);
        MB2_HD inline uint32_t removeMin();
        MB2_HD inline void decreaseCost(uint32_t poly, float cost);

        // moves poly up from heap slot idx to where its cost belongs
        MB2_HD inline void siftUp(CountT idx, uint32_t poly, float cost);
    };

    struct AliasEntry {
        float tau;
        uint32_t alias;
    };

    math::Vector3 *vertices;
    uint32_t *triIndices;
    uint32_t *triAdjacency;
    AliasEntry *triSampleAliasTable;
    uint32_t numVerts;
    uint32_t numTris;

    MB2_HD inline math::Vector3 samplePointAndPoly(RandKey rnd, uint32_t *out_poly);
    MB2_HD inline math::Vector3 samplePoint(RandKey rnd);

    MB2_HD inline void getTriangleVertices(uint32_t tri_idx,
                                           math::Vector3 *out_a,
                                           math::Vector3 *out_b,
                                           math::Vector3 *out_c);

    struct BFSState {
        uint32_t *queue;
        bool *visited;
    };

    template <typename Fn>
    MB2_HD inline void bfsFromPoly(uint32_t poly, BFSState bfs_state, Fn &&fn);

    struct DijkstrasState {
        float *distances;
        math::Vector3 *entryPoints;
        uint32_t *heap;
        uint32_t *heapIndex;
    };

    template <typename Fn>
    MB2_HD inline void dijkstrasFromPoly(uint32_t start_poly,
                                         math::Vector3 start_pos,
                                         DijkstrasState dijkstras_state,
                                         Fn &&fn);

    static inline Navmesh initFromPolygons(math::Vector3 *poly_vertices,
                                           uint32_t *poly_idxs,
                                           uint32_t *poly_idx_offsets,
                                           uint32_t *poly_sizes,
                                           uint32_t num_verts,
                                           uint32_t num_polys);

    static constexpr inline uint32_t sentinel = 0xFFFF'FFFF;

    // ---- construction into caller storage (initFromPolygons and the host builder,
    // mb2_navmesh_create, share it) ------------------------------------------------------
    struct EdgeSlot {
        uint32_t vertA;       // sentinel: empty
        uint32_t vertB;
        uint32_t ownerTri;
        uint32_t ownerEdge;
    };

    // triangles of a polygon soup (sum of size - 2); false if a polygon has fewer than 3
    static MB2_HD inline bool countTriangles(const uint32_t *poly_sizes, uint32_t num_polys,
                                             uint32_t *out_num_tris);

    // out's four arrays are caller storage for numVerts / numTris entries; scratch:
    // weights [numTris], stacks [2 numTris], edges [3 numTris]
    static MB2_HD inline void buildArrays(const math::Vector3 *poly_vertices,
                                          const uint32_t *poly_idxs,
                                          const uint32_t *poly_idx_offsets,
                                          const uint32_t *poly_sizes,
                                          uint32_t num_polys,
                                          Navmesh out,
                                          float *weights,
                                          uint32_t *stacks,
                                          EdgeSlot *edges);
};

static_assert(sizeof(Navmesh) == 40, "Navmesh layout (reference: navmesh.hpp:9-31)");
static_assert(sizeof(Navmesh::AliasEntry) == 8, "AliasEntry layout");
#ifndef __CUDACC_RTC__
// field offsets: checked by the host compilers (NVRTC has no offsetof); the layout is the same
static_assert(offsetof(Navmesh, vertices) == 0 && offsetof(Navmesh, triIndices) == 8 &&
              offsetof(Navmesh, triAdjacency) == 16 && offsetof(Navmesh, triSampleAliasTable) == 24 &&
              offsetof(Navmesh, numVerts) == 32 && offsetof(Navmesh, numTris) == 36,
              "Navmesh field offsets");
static_assert(offsetof(Navmesh::AliasEntry, alias) == 4,
              "AliasEntry layout");
#endif

// ---- priority queue -----------------------------------------------------------------------

void Navmesh::PathFindQueue::siftUp(CountT idx, uint32_t poly, float cost)
{
    while (idx != 0) {
        const CountT parent = (idx - 1) / 2;
        const uint32_t parent_poly = heap[parent];
        if (costs[parent_poly] <= cost) {
            break;
        }
        heap[idx] = parent_poly;
        heapIndex[parent_poly] = (uint32_t)idx;
        idx = parent;
    }
    heap[idx] = poly;
    heapIndex[poly] = (uint32_t)idx;
}

void Navmesh::PathFindQueue::add(uint32_t poly, float cost)
{
    costs[poly] = cost;
    siftUp(heapSize++, poly, cost);
}

uint32_t Navmesh::PathFindQueue::removeMin()
{
    const uint32_t top = heap[0];
    heapSize -= 1;
    const uint32_t last = heap[heapSize];
    const float last_cost = costs[last];

    CountT idx = 0;
    for (;;) {
        CountT child = 2 * idx + 1;
        if (child >= heapSize) {
            break;
        }
        uint32_t child_poly = heap[child];
        float child_cost = costs[child_poly];
        if (child + 1 < heapSize) {
            const uint32_t right_poly = heap[child + 1];
            const float right_cost = costs[right_poly];
            if (right_cost < child_cost) {
                child += 1;
                child_poly = right_poly;
                child_cost = right_cost;
            }
        }
        if (last_cost < child_cost) {
            break;
        }
        heap[idx] = child_poly;
        heapIndex[child_poly] = (uint32_t)idx;
        idx = child;
    }
    heap[idx] = last;
    heapIndex[last] = (uint32_t)idx;

    heapIndex[top] = sentinel;
    return top;
}

void Navmesh::PathFindQueue::decreaseCost(uint32_t poly, float cost)
{
    costs[poly] = cost;
    siftUp((CountT)heapIndex[poly], poly, cost);
}

// ---- queries ------------------------------------------------------------------------------

void Navmesh::getTriangleVertices(uint32_t tri_idx,
                                  math::Vector3 *out_a,
                                  math::Vector3 *out_b,
                                  math::Vector3 *out_c)
{
    const uint32_t *idx = triIndices + 3 * tri_idx;
    *out_a = navmeshRO::ldVec3(vertices + navmeshRO::ld(idx));
    *out_b = navmeshRO::ldVec3(vertices + navmeshRO::ld(idx + 1));
    *out_c = navmeshRO::ldVec3(vertices + navmeshRO::ld(idx + 2));
}

math::Vector3 Navmesh::samplePointAndPoly(RandKey rnd, uint32_t *out_poly)
{
    using namespace math;

    const RandKey row_key = rand::split_i(rnd, 0);
    const RandKey alias_key = rand::split_i(rnd, 1);
    const RandKey bary_key = rand::split_i(rnd, 2);

    const uint32_t row = (uint32_t)rand::sampleI32(row_key, 0, (int32_t)numTris);
    const float p = rand::sampleUniform(alias_key);
    const float tau = navmeshRO::ld(&triSampleAliasTable[row].tau);
    const uint32_t tri = p < tau ? row : navmeshRO::ld(&triSampleAliasTable[row].alias);
    *out_poly = tri;

    Vector3 a, b, c;
    getTriangleVertices(tri, &a, &b, &c);

    Vector2 uv = rand::sample2xUniform(bary_key);
    if (uv.x + uv.y > 1.f) {
        uv.x = 1.f - uv.x;
        uv.y = 1.f - uv.y;
    }
    const float w = 1.f - uv.x - uv.y;
    // products and sums rounded one by one: the engine compiles without FMA contraction
    return a * uv.x + b * uv.y + c * w;
}

math::Vector3 Navmesh::samplePoint(RandKey rnd)
{
    uint32_t poly;
    return samplePointAndPoly(rnd, &poly);
}

template <typename Fn>
MADRONA_ALWAYS_INLINE void Navmesh::bfsFromPoly(uint32_t start_poly, BFSState bfs_state, Fn &&fn)
{
    ArrayQueue<uint32_t> queue(bfs_state.queue, numTris);
    bool *visited = bfs_state.visited;
    utils::zeroN<bool>(visited, numTris);

    queue.add(start_poly);
    visited[start_poly] = true;

    while (!queue.isEmpty()) {
        const uint32_t poly = queue.remove();
        if (!fn(poly)) {
            continue;
        }
        MB2_NAVMESH_UNROLL
        for (int i = 0; i < 3; i++) {
            const uint32_t nbr = navmeshRO::ld(triAdjacency + 3 * poly + i);
            if (nbr != sentinel && !visited[nbr]) {
                queue.add(nbr);
                visited[nbr] = true;
            }
        }
    }
}

template <typename Fn>
MADRONA_ALWAYS_INLINE void Navmesh::dijkstrasFromPoly(uint32_t start_poly,
                                                      math::Vector3 start_pos,
                                                      DijkstrasState st,
                                                      Fn &&fn)
{
    using namespace math;

    float *distances = st.distances;
    Vector3 *entry_points = st.entryPoints;
    PathFindQueue queue { distances, st.heap, st.heapIndex, 0 };
    utils::fillN<uint32_t>(queue.heapIndex, sentinel, numTris);
    utils::fillN<float>(distances, FLT_MAX, numTris);

    entry_points[start_poly] = start_pos;
    queue.add(start_poly, 0.f);

    while (queue.heapSize > 0) {
        const uint32_t poly = queue.removeMin();
        const Vector3 cur = entry_points[poly];
        const float dist = distances[poly];

        fn(poly, cur, dist);

        Vector3 a, b, c;
        getTriangleVertices(poly, &a, &b, &c);
        const Vector3 mids[3] = { (a + b) / 2.f, (b + c) / 2.f, (c + a) / 2.f };

        MB2_NAVMESH_UNROLL
        for (int i = 0; i < 3; i++) {
            const uint32_t nbr = navmeshRO::ld(triAdjacency + 3 * poly + i);
            if (nbr == sentinel) {
                continue;
            }
            const float new_dist = dist + cur.distance(mids[i]);
            if (new_dist >= distances[nbr]) {
                continue;
            }
            entry_points[nbr] = mids[i];
            if (queue.heapIndex[nbr] == sentinel) {
                queue.add(nbr, new_dist);
            } else {
                queue.decreaseCost(nbr, new_dist);
            }
        }
    }
}

// ---- construction -------------------------------------------------------------------------

bool Navmesh::countTriangles(const uint32_t *poly_sizes, uint32_t num_polys, uint32_t *out_num_tris)
{
    uint32_t n = 0;
    for (uint32_t i = 0; i < num_polys; i++) {
        if (poly_sizes[i] < 3) {
            return false;
        }
        n += poly_sizes[i] - 2;
    }
    *out_num_tris = n;
    return true;
}

void Navmesh::buildArrays(const math::Vector3 *poly_vertices,
                          const uint32_t *poly_idxs,
                          const uint32_t *poly_idx_offsets,
                          const uint32_t *poly_sizes,
                          uint32_t num_polys,
                          Navmesh out,
                          float *weights,
                          uint32_t *stacks,
                          EdgeSlot *edges)
{
    using namespace math;
    const uint32_t T = out.numTris;

    utils::copyN<Vector3>(out.vertices, poly_vertices, out.numVerts);

    // fan every polygon from its first index; weight = twice the triangle's area
    float weight_sum = 0.f;
    uint32_t tri = 0;
    for (uint32_t p = 0; p < num_polys; p++) {
        const uint32_t base = poly_idx_offsets[p];
        const uint32_t ia = poly_idxs[base];
        for (uint32_t k = 1; k + 1 < poly_sizes[p]; k++) {
            const uint32_t ib = poly_idxs[base + k];
            const uint32_t ic = poly_idxs[base + k + 1];
            out.triIndices[3 * tri] = ia;
            out.triIndices[3 * tri + 1] = ib;
            out.triIndices[3 * tri + 2] = ic;
            const Vector3 a = poly_vertices[ia];
            const Vector3 e1 = poly_vertices[ib] - a;
            const Vector3 e2 = poly_vertices[ic] - a;
            const float w = cross(e1, e2).length();
            weights[tri] = w;
            weight_sum += w;
            tri += 1;
        }
    }

    // Vose's alias table: "under" entries (normalised weight below 1) borrow the rest of
    // their slot from an "over" entry, both taken from the top of their stacks
    uint32_t *under = stacks;
    uint32_t *over = stacks + T;
    uint32_t num_under = 0, num_over = 0;
    for (uint32_t t = 0; t < T; t++) {
        const float w = weights[t] * float(T) / weight_sum;
        weights[t] = w;
        if (w < 1.f) {
            under[num_under++] = t;
        } else {
            over[num_over++] = t;
        }
    }
    while (num_under != 0 && num_over != 0) {
        const uint32_t u = under[--num_under];
        const uint32_t o = over[--num_over];
        out.triSampleAliasTable[u] = AliasEntry { weights[u], o };
        const float rest = (weights[o] + weights[u]) - 1.f;
        weights[o] = rest;
        if (rest < 1.f) {
            under[num_under++] = o;
        } else {
            over[num_over++] = o;
        }
    }
    for (uint32_t i = 0; i < num_under; i++) {
        out.triSampleAliasTable[under[i]] = AliasEntry { 1.f, under[i] };
    }
    for (uint32_t i = 0; i < num_over; i++) {
        out.triSampleAliasTable[over[i]] = AliasEntry { 1.f, over[i] };
    }

    // adjacency: the first triangle with an edge owns it; each later one links itself to
    // the owner and points the owner at itself (so a non-manifold edge's owner ends up
    // linked to its last visitor).  Open addressing over 3T slots, linear probing.
    const uint32_t num_slots = 3 * T;
    for (uint32_t i = 0; i < num_slots; i++) {
        out.triAdjacency[i] = sentinel;
        edges[i] = EdgeSlot { sentinel, sentinel, sentinel, 0 };
    }
    for (uint32_t t = 0; t < T; t++) {
        for (uint32_t e = 0; e < 3; e++) {
            uint32_t va = out.triIndices[3 * t + e];
            uint32_t vb = out.triIndices[3 * t + (e == 2 ? 0 : e + 1)];
            if (vb < va) {
                const uint32_t s = va;
                va = vb;
                vb = s;
            }
            uint32_t slot = utils::u32mulhi(utils::int32Hash(va * 0x9E3779B1u ^ utils::int32Hash(vb)),
                                            num_slots);
            while (edges[slot].vertA != sentinel &&
                   (edges[slot].vertA != va || edges[slot].vertB != vb)) {
                slot = slot + 1 == num_slots ? 0 : slot + 1;
            }
            EdgeSlot &s = edges[slot];
            if (s.vertA == sentinel) {
                s = EdgeSlot { va, vb, t, e };
            } else {
                out.triAdjacency[3 * t + e] = s.ownerTri;
                out.triAdjacency[3 * s.ownerTri + s.ownerEdge] = t;
            }
        }
    }
}

Navmesh Navmesh::initFromPolygons(math::Vector3 *poly_vertices,
                                  uint32_t *poly_idxs,
                                  uint32_t *poly_idx_offsets,
                                  uint32_t *poly_sizes,
                                  uint32_t num_verts,
                                  uint32_t num_polys)
{
    using namespace math;
    Navmesh none { nullptr, nullptr, nullptr, nullptr, 0, 0 };
    uint32_t T = 0;
    if (!countTriangles(poly_sizes, num_polys, &T)) {
#ifdef MADRONA_GPU_MODE
        mwGPU::raiseError(mb2::ErrNavmeshPolygon);
#endif
        return none;
    }

    Navmesh out;
    out.numVerts = num_verts;
    out.numTris = T;
    out.vertices = (Vector3 *)rawAlloc(sizeof(Vector3) * num_verts);
    out.triIndices = (uint32_t *)rawAlloc(sizeof(uint32_t) * 3 * T);
    out.triAdjacency = (uint32_t *)rawAlloc(sizeof(uint32_t) * 3 * T);
    out.triSampleAliasTable = (AliasEntry *)rawAlloc(sizeof(AliasEntry) * T);
#ifdef MADRONA_GPU_MODE
    float *weights = (float *)mwGPU::tmpArenaAlloc(sizeof(float) * T);
    uint32_t *stacks = (uint32_t *)mwGPU::tmpArenaAlloc(sizeof(uint32_t) * 2 * T);
    EdgeSlot *edges = (EdgeSlot *)mwGPU::tmpArenaAlloc(sizeof(EdgeSlot) * 3 * T);
#else
    float *weights = (float *)malloc(sizeof(float) * T);
    uint32_t *stacks = (uint32_t *)malloc(sizeof(uint32_t) * 2 * T);
    EdgeSlot *edges = (EdgeSlot *)malloc(sizeof(EdgeSlot) * 3 * T);
#endif
    const bool ok = out.vertices && out.triIndices && out.triAdjacency && out.triSampleAliasTable &&
                    weights && stacks && edges;
    if (ok) {
        buildArrays(poly_vertices, poly_idxs, poly_idx_offsets, poly_sizes, num_polys, out,
                    weights, stacks, edges);
    }
#ifndef MADRONA_GPU_MODE
    free(weights);
    free(stacks);
    free(edges);
    if (!ok) {
        free(out.vertices);
        free(out.triIndices);
        free(out.triAdjacency);
        free(out.triSampleAliasTable);
    }
#endif
    return ok ? out : none;
}

}
