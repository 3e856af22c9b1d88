// Floor plans of the navmesh fixture: a seeded variant of a 6 x 6 grid of unit cells on
// z = 0, as a polygon soup for Navmesh::initFromPolygons.  Plain C++ with exact float
// coordinates (multiples of 0.5), so host and device, and sims/navmesh_plan.py, build the
// same soup bit for bit.
//   * polygon 0 is a hexagon over cells (0,0) and (1,0) whose fan starts with a
//     zero-area triangle;
//   * each other cell is removed (1 in 8), a quad, or (1 in 8) a pentagon with a vertex
//     in the middle of its +x edge; column 4 is a wall with at most one door, so a plan
//     may fall apart into islands;
//   * a vertical fin triangle on the edge between cells (2,1) and (2,2), which are always
//     quads: an edge shared by three triangles;
//   * one separate weight-2 triangle per pentagon (always an island).  Every polygon kind
//     then has as many triangles as its summed weights, so weights sum to the triangle
//     count and every unit triangle's normalised weight is exactly 1.
#pragma once
#include <cstdint>

namespace navmesh {

constexpr uint32_t kGrid = 6;
constexpr uint32_t kWallColumn = 4;
constexpr uint32_t kLattice = (kGrid + 1) * (kGrid + 1);
constexpr uint32_t kMaxPlanVerts = kLattice + 1 + kGrid * kGrid * 4;
constexpr uint32_t kMaxPlanPolys = kGrid * kGrid * 2 + 4;
constexpr uint32_t kMaxPlanIdxs = kMaxPlanPolys * 6;
// the plan every world shares through Config
constexpr uint32_t kSharedPlanSeed = 0x5eedu;

struct Plan {
    float xyz[kMaxPlanVerts * 3];
    uint32_t idxs[kMaxPlanIdxs];
    uint32_t offsets[kMaxPlanPolys];
    uint32_t sizes[kMaxPlanPolys];
    uint32_t numVerts;
    uint32_t numIdxs;
    uint32_t numPolys;
};

inline uint32_t planHash(uint32_t seed, uint32_t i)
{
    uint32_t x = seed * 0x9E3779B9u + i * 0x85EBCA6Bu + 0x165667B1u;
    x ^= x >> 16;
    x *= 0x7feb352du;
    x ^= x >> 15;
    x *= 0x846ca68bu;
    x ^= x >> 16;
    return x;
}

struct PlanWriter {
    Plan &p;

    uint32_t vert(float x, float y, float z)
    {
        p.xyz[3 * p.numVerts] = x;
        p.xyz[3 * p.numVerts + 1] = y;
        p.xyz[3 * p.numVerts + 2] = z;
        return p.numVerts++;
    }

    void poly(const uint32_t *idxs, uint32_t n)
    {
        p.offsets[p.numPolys] = p.numIdxs;
        p.sizes[p.numPolys] = n;
        p.numPolys += 1;
        for (uint32_t i = 0; i < n; i++) {
            p.idxs[p.numIdxs++] = idxs[i];
        }
    }
};

inline uint32_t latticeIdx(uint32_t i, uint32_t j) { return j * (kGrid + 1) + i; }

// bad_polygon: append a 2-vertex polygon (initFromPolygons must reject the plan)
inline void makePlan(uint32_t seed, uint32_t bad_polygon, Plan &p)
{
    p.numVerts = 0;
    p.numIdxs = 0;
    p.numPolys = 0;
    PlanWriter w { p };
    for (uint32_t j = 0; j <= kGrid; j++) {
        for (uint32_t i = 0; i <= kGrid; i++) {
            w.vert((float)i, (float)j, 0.f);
        }
    }
    const uint32_t apex = w.vert(2.5f, 2.f, 1.f);

    const uint32_t hex[6] = { latticeIdx(0, 0), latticeIdx(1, 0), latticeIdx(2, 0),
                              latticeIdx(2, 1), latticeIdx(1, 1), latticeIdx(0, 1) };
    w.poly(hex, 6);

    const uint32_t door = planHash(seed, 1000) % (kGrid + 2);
    uint32_t num_pentagons = 0;
    for (uint32_t j = 0; j < kGrid; j++) {
        for (uint32_t i = 0; i < kGrid; i++) {
            if (j == 0 && i < 2) {
                continue;
            }
            const uint32_t a = latticeIdx(i, j), b = latticeIdx(i + 1, j);
            const uint32_t c = latticeIdx(i + 1, j + 1), d = latticeIdx(i, j + 1);
            const bool fixed = i == 2 && (j == 1 || j == 2);
            if (!fixed) {
                if (i == kWallColumn && j != door) {
                    continue;
                }
                const uint32_t r = planHash(seed, j * kGrid + i) % 8;
                if (r == 0) {
                    continue;
                }
                if (r == 1) {
                    const uint32_t m = w.vert((float)(i + 1), (float)j + 0.5f, 0.f);
                    const uint32_t pent[5] = { a, b, m, c, d };
                    w.poly(pent, 5);
                    num_pentagons += 1;
                    continue;
                }
            }
            const uint32_t quad[4] = { a, b, c, d };
            w.poly(quad, 4);
        }
    }

    const uint32_t fin[3] = { latticeIdx(2, 2), latticeIdx(3, 2), apex };
    w.poly(fin, 3);

    for (uint32_t k = 0; k < num_pentagons; k++) {
        const float x = (float)(kGrid + 1), y = (float)(2 * k);
        const uint32_t v0 = w.vert(x, y, 0.f);
        const uint32_t v1 = w.vert(x + 2.f, y, 0.f);
        const uint32_t v2 = w.vert(x, y + 1.f, 0.f);
        const uint32_t tri[3] = { v0, v1, v2 };
        w.poly(tri, 3);
    }

    if (bad_polygon) {
        const uint32_t two[2] = { latticeIdx(0, 0), latticeIdx(1, 0) };
        w.poly(two, 2);
    }
}

}
