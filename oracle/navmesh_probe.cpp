// TEST INFRASTRUCTURE ONLY: navmesh equivalence probe.  The same source is built against the
// reference (include/madrona/navmesh.hpp + src/common/navmesh.cpp, -DPROBE_REF) and against
// the engine's device headers (madrona_b200/device/madrona/navmesh.hpp, whose
// Navmesh::buildArrays the host builder mb2_navmesh_create runs); tests/test_navmesh.py
// requires the two outputs to be identical.  For many polygon soups -- the fixture's floor
// plans, jittered lattices, random convex polygons sharing edges, repeated vertex indices,
// single triangles -- it prints the four arrays, samplePointAndPoly results, and the BFS and
// Dijkstra callback sequences from every start triangle; then the utils functions.
// Built by oracle/navmesh.mk.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include <madrona/navmesh.hpp>
#include <madrona/utils.hpp>
#include <madrona/memory.hpp>

#include "../sims/navmesh/plan.hpp"

using namespace madrona;
using namespace madrona::math;

static uint32_t fb(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
}

struct Rng {
    uint64_t s;
    uint32_t next()
    {
        s = s * 6364136223846793005ull + 1442695040888963407ull;
        return (uint32_t)(s >> 32);
    }
    // [0, 1) with 24 random bits
    float unit() { return (float)(next() >> 8) * (1.f / 16777216.f); }
};

struct Soup {
    std::vector<float> xyz;
    std::vector<uint32_t> idx, off, sizes;

    uint32_t vert(float x, float y, float z)
    {
        xyz.push_back(x);
        xyz.push_back(y);
        xyz.push_back(z);
        return (uint32_t)(xyz.size() / 3 - 1);
    }
    void poly(std::initializer_list<uint32_t> l)
    {
        off.push_back((uint32_t)idx.size());
        sizes.push_back((uint32_t)l.size());
        for (uint32_t v : l) idx.push_back(v);
    }
    void polyv(const std::vector<uint32_t> &l)
    {
        off.push_back((uint32_t)idx.size());
        sizes.push_back((uint32_t)l.size());
        for (uint32_t v : l) idx.push_back(v);
    }
};

static void probeSoup(const char *name, Soup &s, uint32_t num_samples)
{
    const uint32_t nv = (uint32_t)(s.xyz.size() / 3), np = (uint32_t)s.sizes.size();
    Navmesh m = Navmesh::initFromPolygons((Vector3 *)s.xyz.data(), s.idx.data(), s.off.data(), s.sizes.data(),
                                          nv, np);
    const uint32_t T = m.numTris;
    printf("soup %s V %u T %u\n", name, m.numVerts, T);
    for (uint32_t i = 0; i < m.numVerts; i++) {
        printf("v %08x %08x %08x\n", fb(m.vertices[i].x), fb(m.vertices[i].y), fb(m.vertices[i].z));
    }
    for (uint32_t t = 0; t < T; t++) {
        printf("t %u %u %u | %u %u %u | %08x %u\n", m.triIndices[3 * t], m.triIndices[3 * t + 1],
               m.triIndices[3 * t + 2], m.triAdjacency[3 * t], m.triAdjacency[3 * t + 1],
               m.triAdjacency[3 * t + 2], fb(m.triSampleAliasTable[t].tau), m.triSampleAliasTable[t].alias);
    }
    for (uint32_t k = 0; k < num_samples; k++) {
        RandKey key = rand::split_i(rand::initKey(0xABCDu + T, k), k * 7u);
        uint32_t p = 0;
        Vector3 x = m.samplePointAndPoly(key, &p);
        Vector3 y = m.samplePoint(key);
        printf("s %u %08x %08x %08x %08x\n", p, fb(x.x), fb(x.y), fb(x.z), fb(y.x) ^ fb(y.y) ^ fb(y.z));
    }

    std::vector<uint32_t> queue(T + 1), heap(T + 1), heap_idx(T + 1);
    std::unique_ptr<bool[]> visited(new bool[T + 1]);
    std::vector<float> dist(T + 1);
    std::vector<Vector3> entry(T + 1);
    for (uint32_t start = 0; start < T; start++) {
        printf("b %u:", start);
        m.bfsFromPoly(start, Navmesh::BFSState { queue.data(), visited.get() }, [&](uint32_t t) {
            printf(" %u", t);
            return t == start || (t * 3 + start) % 4 != 0;
        });
        printf("\n");

        Vector3 a, b, c;
        m.getTriangleVertices(start, &a, &b, &c);
        const Vector3 from = (a + b + c) / 3.f;
        printf("d %u:", start);
        m.dijkstrasFromPoly(start, from,
            Navmesh::DijkstrasState { dist.data(), entry.data(), heap.data(), heap_idx.data() },
            [&](uint32_t t, Vector3 e, float d) {
                printf(" %u/%08x/%08x%08x%08x", t, fb(d), fb(e.x), fb(e.y), fb(e.z));
            });
        printf("\n");
    }
}

static void fixturePlan(uint32_t seed, uint32_t num_samples)
{
    static navmesh::Plan plan;
    navmesh::makePlan(seed, 0, plan);
    printf("plan %u V %u P %u I %u\n", seed, plan.numVerts, plan.numPolys, plan.numIdxs);
    for (uint32_t i = 0; i < 3 * plan.numVerts; i++) printf(" %08x", fb(plan.xyz[i]));
    printf("\n");
    for (uint32_t p = 0; p < plan.numPolys; p++) {
        printf(" %u/%u", plan.offsets[p], plan.sizes[p]);
    }
    printf("\n");
    for (uint32_t i = 0; i < plan.numIdxs; i++) printf(" %u", plan.idxs[i]);
    printf("\n");
    Soup s;
    s.xyz.assign(plan.xyz, plan.xyz + 3 * plan.numVerts);
    s.idx.assign(plan.idxs, plan.idxs + plan.numIdxs);
    s.off.assign(plan.offsets, plan.offsets + plan.numPolys);
    s.sizes.assign(plan.sizes, plan.sizes + plan.numPolys);
    char name[32];
    snprintf(name, sizeof(name), "plan%u", seed);
    probeSoup(name, s, num_samples);
}

// jittered lattice: quads, some removed, some 2-cell hexagons; random float coordinates
static void latticeSoup(uint32_t seed, uint32_t n)
{
    Rng r { seed * 0x9E3779B97F4A7C15ull + 1 };
    Soup s;
    for (uint32_t j = 0; j <= n; j++) {
        for (uint32_t i = 0; i <= n; i++) {
            s.vert((float)i + 0.3f * r.unit(), (float)j + 0.3f * r.unit(), 0.25f * r.unit());
        }
    }
    auto L = [n](uint32_t i, uint32_t j) { return j * (n + 1) + i; };
    for (uint32_t j = 0; j < n; j++) {
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t k = r.next() % 6;
            if (k == 0) continue;
            if (k == 1 && i + 2 <= n && j % 2 == 0) {
                s.poly({ L(i, j), L(i + 1, j), L(i + 2, j), L(i + 2, j + 1), L(i + 1, j + 1), L(i, j + 1) });
                i += 1;
                continue;
            }
            s.poly({ L(i, j), L(i + 1, j), L(i + 1, j + 1), L(i, j + 1) });
        }
    }
    char name[32];
    snprintf(name, sizeof(name), "lattice%u", seed);
    probeSoup(name, s, 1000);
}

// random convex polygons (vertices on circles, in angle order); each polygon but the first
// starts with an edge of an earlier one, reversed, so edges are shared by two or more
// polygons (the borrowed edge can make such a polygon non-convex)
static void convexSoup(uint32_t seed, uint32_t num_polys)
{
    Rng r { seed * 0xD1B54A32D192ED03ull + 7 };
    Soup s;
    std::vector<std::pair<uint32_t, uint32_t>> edges;
    for (uint32_t p = 0; p < num_polys; p++) {
        const uint32_t k = 3 + r.next() % 6;
        const float cx = 10.f * r.unit(), cy = 10.f * r.unit(), rad = 0.5f + 2.f * r.unit();
        std::vector<uint32_t> loop;
        uint32_t first = 0;
        if (!edges.empty()) {
            const auto e = edges[r.next() % edges.size()];
            loop.push_back(e.second);
            loop.push_back(e.first);
            first = 2;
        }
        // points on a circle in angle order through the rational parametrisation
        // ((1 - t^2), 2t) / (1 + t^2) with t increasing: a convex loop
        float t = -4.f;
        for (uint32_t v = first; v < k; v++) {
            t += (0.1f + r.unit()) * 8.f / (float)k;
            const float d = 1.f + t * t;
            loop.push_back(s.vert(cx + rad * (1.f - t * t) / d, cy + rad * 2.f * t / d, 0.1f * r.unit()));
        }
        for (size_t i = 0; i < loop.size(); i++) {
            edges.push_back({ loop[i], loop[(i + 1) % loop.size()] });
        }
        s.polyv(loop);
    }
    char name[32];
    snprintf(name, sizeof(name), "convex%u", seed);
    probeSoup(name, s, 1000);
}

static void utilsProbe()
{
    uint32_t store[5];
    ArrayQueue<uint32_t> q(store, 5);
    printf("queue cap %u empty %d\n", q.capacity(), (int)q.isEmpty());
    uint32_t next = 0;
    Rng r { 99 };
    for (int i = 0; i < 200; i++) {
        const uint32_t op = r.next() % 3;
        if (op != 0 && next < 1000) {
            q.add(next++);
            printf(" +%u", next - 1);
        }
        if (op == 0 && !q.isEmpty()) {
            printf(" -%u", q.remove());
        }
        if (i % 37 == 36) {
            q.clear();
            printf(" c%d", (int)q.isEmpty());
        }
    }
    printf("\n");

    printf("hash");
    for (uint32_t i = 0; i < 4096; i++) printf(" %08x", utils::int32Hash(i * 2654435761u));
    printf("\n");
    printf("pow2");
    for (uint64_t v = 1; v <= (1ull << 31); v = v < 70 ? v + 1 : v * 3 / 2 + 1) {
        const uint32_t v32 = (uint32_t)v;
        printf(" %u:%u:%u:%llu:%llu:%d:%d", v32, utils::int32NextPow2(v32), utils::int32Log2(v32),
               (unsigned long long)utils::int64NextPow2(v), (unsigned long long)utils::int64Log2(v),
               (int)utils::isPower2(v32), (int)utils::isPower2((uint64_t)v));
    }
    printf(" %llu", (unsigned long long)utils::int64Log2(0xFFFFFFFFFFFFull));
    printf("\n");
    alignas(256) static char buf[1024];
    printf("align");
    for (uintptr_t a = 1; a <= 256; a *= 2) {
        for (int o = 0; o < 40; o += 3) {
            printf(" %lu:%ld", (unsigned long)utils::alignPtrOffset(buf + o, a),
                   (long)((char *)utils::alignPtr(buf + o, a) - buf));
        }
    }
    printf("\n");
    int64_t sizes[5] = { 10, 1, 300, 0, 77 };
    int64_t offs[4] = {};
    for (int64_t al : { 1, 8, 64, 256 }) {
        const int64_t total = utils::computeBufferOffsets(Span<const int64_t>(sizes, 5), Span<int64_t>(offs, 4), al);
        printf("offsets %ld: %ld %ld %ld %ld -> %ld\n", (long)al, (long)offs[0], (long)offs[1], (long)offs[2],
               (long)offs[3], (long)total);
    }
    uint32_t a[9] = { 1, 2, 3, 4, 5, 6, 7, 8, 9 }, b[9] = {};
    utils::copyN<uint32_t>(b, a, 7);
    utils::fillN<uint32_t>(a, 42u, 4);
    utils::zeroN<uint32_t>(a + 6, 2);
    printf("copy");
    for (int i = 0; i < 9; i++) printf(" %u/%u", a[i], b[i]);
    printf("\n");
}

int main()
{
    fixturePlan(navmesh::kSharedPlanSeed, 3000);
    for (uint32_t seed = 0; seed < 12; seed++) fixturePlan(seed, 200);
    for (uint32_t seed = 1; seed <= 6; seed++) latticeSoup(seed, 4 + seed);
    for (uint32_t seed = 1; seed <= 8; seed++) convexSoup(seed, 6 + 4 * seed);

    Soup repeated;
    for (int i = 0; i < 5; i++) repeated.vert((float)(i % 3), (float)(i / 2), 0.5f * (float)i);
    repeated.poly({ 0, 1, 1, 2 });
    repeated.poly({ 0, 0, 1 });
    repeated.poly({ 2, 1, 3, 4, 4 });
    repeated.poly({ 3, 2, 1 });
    probeSoup("repeated", repeated, 500);

    Soup single;
    single.vert(0.f, 0.f, 0.f);
    single.vert(1.5f, 0.25f, 0.f);
    single.vert(0.125f, 2.f, 0.5f);
    single.poly({ 0, 1, 2 });
    probeSoup("single", single, 500);

    Soup flat;
    flat.vert(0.f, 0.f, 0.f);
    flat.vert(1.f, 1.f, 1.f);
    flat.vert(2.f, 2.f, 2.f);
    flat.poly({ 0, 1, 2 });
    flat.poly({ 2, 1, 0 });
    probeSoup("zeroarea", flat, 100);

    utilsProbe();
    return 0;
}
