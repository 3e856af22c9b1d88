// navmesh_host.cpp -- the host navmesh builder: one polygon soup in, the four arrays of a
// madrona::Navmesh out (the reference's host Navmesh::initFromPolygons, src/common/
// navmesh.cpp), uploaded to the GPU once, so that worlds sharing one floor plan share one
// mesh instead of building thousands of copies on the device.  The arrays come from the
// same Navmesh::buildArrays the device initFromPolygons runs; this translation unit is
// compiled with -ffp-contract=off, so they are bit-identical to the reference's.
#include "../../include/madrona_b200.h"
#include "engine.hpp"

#include <madrona/navmesh.hpp>

#include <cuda_runtime.h>
#include <cstring>
#include <string>
#include <vector>

namespace mb2 {
namespace {

using madrona::Navmesh;
using madrona::math::Vector3;

struct NavmeshBundle {
    std::vector<Vector3> vertices;
    std::vector<uint32_t> triIndices;
    std::vector<uint32_t> triAdjacency;
    std::vector<Navmesh::AliasEntry> aliasTable;
    Navmesh deviceView {};
    void *deviceBlock = nullptr;
    int gpu = -1;
};

}
}

using namespace mb2;

extern "C" {

mb2_navmesh *mb2_navmesh_create(const float *vertices_xyz, uint32_t num_verts,
                                const uint32_t *poly_idxs, uint32_t num_idxs,
                                const uint32_t *poly_offsets, const uint32_t *poly_sizes,
                                uint32_t num_polys, int gpu_id)
{
    const std::string where = "mb2_navmesh_create: ";
    if (!vertices_xyz || !poly_idxs || !poly_offsets || !poly_sizes) {
        setError(where + "null input array");
        return nullptr;
    }
    if (num_polys == 0) {
        setError(where + "no polygons");
        return nullptr;
    }
    uint64_t num_tris = 0;
    for (uint32_t p = 0; p < num_polys; p++) {
        if (poly_sizes[p] < 3) {
            setError(where + "polygon " + std::to_string(p) + " has " + std::to_string(poly_sizes[p]) +
                     " vertices (at least 3 needed)");
            return nullptr;
        }
        if ((uint64_t)poly_offsets[p] + poly_sizes[p] > num_idxs) {
            setError(where + "polygon " + std::to_string(p) + " runs past the index array (offset " +
                     std::to_string(poly_offsets[p]) + " + size " + std::to_string(poly_sizes[p]) + " > " +
                     std::to_string(num_idxs) + ")");
            return nullptr;
        }
        for (uint32_t k = 0; k < poly_sizes[p]; k++) {
            const uint32_t v = poly_idxs[poly_offsets[p] + k];
            if (v >= num_verts) {
                setError(where + "polygon " + std::to_string(p) + " names vertex " + std::to_string(v) +
                         " of " + std::to_string(num_verts));
                return nullptr;
            }
        }
        num_tris += poly_sizes[p] - 2;
    }
    if (num_tris > 0x3FFFFFFFull) {
        setError(where + "too many triangles");
        return nullptr;
    }
    const uint32_t T = (uint32_t)num_tris;

    auto *b = new NavmeshBundle;
    b->gpu = gpu_id;
    b->vertices.resize(num_verts);
    b->triIndices.resize(3 * (size_t)T);
    b->triAdjacency.resize(3 * (size_t)T);
    b->aliasTable.resize(T);
    std::vector<float> weights(T);
    std::vector<uint32_t> stacks(2 * (size_t)T);
    std::vector<Navmesh::EdgeSlot> edges(3 * (size_t)T);
    Navmesh host { b->vertices.data(), b->triIndices.data(), b->triAdjacency.data(), b->aliasTable.data(),
                   num_verts, T };
    Navmesh::buildArrays((const Vector3 *)vertices_xyz, poly_idxs, poly_offsets, poly_sizes, num_polys, host,
                         weights.data(), stacks.data(), edges.data());

    if (gpu_id >= 0) {
        const size_t sz[4] = { sizeof(Vector3) * num_verts, sizeof(uint32_t) * 3 * (size_t)T,
                               sizeof(uint32_t) * 3 * (size_t)T, sizeof(Navmesh::AliasEntry) * T };
        const void *src[4] = { b->vertices.data(), b->triIndices.data(), b->triAdjacency.data(),
                               b->aliasTable.data() };
        size_t off[4], total = 0;
        for (int i = 0; i < 4; i++) {
            off[i] = total;
            total += (sz[i] + 255) & ~(size_t)255;
        }
        std::vector<char> staged(total, 0);
        for (int i = 0; i < 4; i++) {
            if (sz[i]) memcpy(staged.data() + off[i], src[i], sz[i]);
        }
        if (cudaSetDevice(gpu_id) != cudaSuccess || cudaMalloc(&b->deviceBlock, total) != cudaSuccess ||
                cudaMemcpy(b->deviceBlock, staged.data(), total, cudaMemcpyHostToDevice) != cudaSuccess) {
            cudaGetLastError();
            setError(where + "device allocation or upload failed");
            if (b->deviceBlock) cudaFree(b->deviceBlock);
            delete b;
            return nullptr;
        }
        char *base = (char *)b->deviceBlock;
        b->deviceView = Navmesh { (Vector3 *)(base + off[0]), (uint32_t *)(base + off[1]),
                                  (uint32_t *)(base + off[2]), (Navmesh::AliasEntry *)(base + off[3]),
                                  num_verts, T };
    }
    return (mb2_navmesh *)b;
}

const void *mb2_navmesh_view(const mb2_navmesh *h)
{
    const NavmeshBundle *b = (const NavmeshBundle *)h;
    if (!b || !b->deviceBlock) return nullptr;
    return &b->deviceView;
}

void mb2_navmesh_host_arrays(const mb2_navmesh *h, mb2_navmesh_arrays *out)
{
    const NavmeshBundle *b = (const NavmeshBundle *)h;
    if (!b) {
        *out = mb2_navmesh_arrays {};
        return;
    }
    *out = mb2_navmesh_arrays { (const float *)b->vertices.data(), b->triIndices.data(), b->triAdjacency.data(),
                                b->aliasTable.data(), (uint32_t)b->vertices.size(),
                                (uint32_t)b->aliasTable.size() };
}

void mb2_navmesh_destroy(mb2_navmesh *h)
{
    NavmeshBundle *b = (NavmeshBundle *)h;
    if (!b) return;
    if (b->deviceBlock) {
        cudaSetDevice(b->gpu);
        cudaFree(b->deviceBlock);
    }
    delete b;
}

}
