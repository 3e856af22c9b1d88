// A Manager-style snippet that traces physics rays through the C++ facade
// (madrona_b200/host/madrona/mw_gpu.hpp, MWCudaExecutor::tracePhysicsRays).  It uploads the
// rays fixture's ObjectManager, builds sims/rays with 4 worlds (seeds 5-8, a respawn every 4
// steps), steps it 5 times, then traces the fixture's 4 x 64 rays in reverse order (world 3's
// last ray first) from its exported columns into its own device buffers and writes the hits,
// entity int32 [n][2], t float [n], normal float [n][3], to a file:
//   facade_physics_rays <rays sim.cpp> <objects file> <output file>
// The objects file is sims/objects.py's write_blob_file: u64 size, u64 relocation count,
// u64 relocations[] (offsets of u64 blob-relative pointers), blob.
#include <madrona/mw_gpu.hpp>

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

extern "C" int cudaMemcpy(void *, const void *, size_t, int);
extern "C" int cudaMalloc(void **, size_t);
extern "C" int cudaFree(void *);
extern "C" int cudaDeviceSynchronize();

struct Config { void *objMgr; uint32_t episodeLen, uniformBodies, variedBodies, pad; };
struct WorldInit { uint32_t seed; };

int main(int argc, char **argv)
{
    if (argc < 4) return 2;
    constexpr uint32_t num_worlds = 4, rays_per_world = 64, n = num_worlds * rays_per_world;

    FILE *f = fopen(argv[2], "rb");
    if (!f) return 3;
    uint64_t size = 0, num_relocs = 0;
    if (fread(&size, 8, 1, f) != 1 || fread(&num_relocs, 8, 1, f) != 1) return 3;
    std::vector<uint64_t> relocs(num_relocs);
    std::vector<unsigned char> blob(size);
    if (fread(relocs.data(), 8, num_relocs, f) != num_relocs || fread(blob.data(), 1, size, f) != size) return 3;
    fclose(f);

    CUcontext ctx = madrona::MWCudaExecutor::initCUDA(0);
    void *dev_blob = nullptr;
    cudaMalloc(&dev_blob, size);
    for (uint64_t where : relocs) {
        uint64_t off;
        memcpy(&off, blob.data() + where, 8);
        off += (uint64_t)(uintptr_t)dev_blob;
        memcpy(blob.data() + where, &off, 8);
    }
    cudaMemcpy(dev_blob, blob.data(), size, 1 /* HtoD */);

    Config cfg { dev_blob, 4, 0, 0, 0 };
    std::vector<WorldInit> inits(num_worlds);
    for (uint32_t i = 0; i < num_worlds; i++) inits[i].seed = 5 + i;
    std::string include = std::string("-I") + argv[1];
    include = include.substr(0, include.rfind('/'));
    const char *sources[] = { argv[1] };
    const char *flags[] = { include.c_str() };
    {
        madrona::MWCudaExecutor exec({
            .worldInitPtr = inits.data(),
            .numWorldInitBytes = sizeof(WorldInit),
            .userConfigPtr = &cfg,
            .numUserConfigBytes = sizeof(Config),
            .numWorldDataBytes = 0,
            .worldDataAlignment = 16,
            .numWorlds = num_worlds,
            .numTaskGraphs = 1,
            .numExportedBuffers = 9,
        }, {
            .userSources = madrona::Span<const char * const>(sources, 1),
            .userCompileFlags = madrona::Span<const char * const>(flags, 1),
        }, ctx);

        madrona::MWCudaLaunchGraph step = exec.buildLaunchGraphAllTaskGraphs();
        for (int i = 0; i < 5; i++) exec.run(step);

        // the fixture's rays (slots 0 - 2: [world][64] origins, directions, max_t), reversed
        std::vector<float> o(n * 3), d(n * 3), m(n), ro(n * 3), rd(n * 3), rm(n);
        cudaMemcpy(o.data(), exec.getExported(0), o.size() * 4, 2 /* DtoH */);
        cudaMemcpy(d.data(), exec.getExported(1), d.size() * 4, 2);
        cudaMemcpy(m.data(), exec.getExported(2), m.size() * 4, 2);
        std::vector<int32_t> world(n);
        for (uint32_t i = 0; i < n; i++) {
            const uint32_t src = n - 1 - i;
            world[i] = (int32_t)(src / rays_per_world);
            for (int c = 0; c < 3; c++) {
                ro[3 * i + c] = o[3 * src + c];
                rd[3 * i + c] = d[3 * src + c];
            }
            rm[i] = m[src];
        }
        void *bufs[7] = {};
        const size_t bytes[7] = { n * 4, n * 12, n * 12, n * 4, n * 8, n * 4, n * 12 };
        const void *host[4] = { world.data(), ro.data(), rd.data(), rm.data() };
        for (int k = 0; k < 7; k++) cudaMalloc(&bufs[k], bytes[k]);
        for (int k = 0; k < 4; k++) cudaMemcpy(bufs[k], host[k], bytes[k], 1 /* HtoD */);
        exec.tracePhysicsRays(madrona_b200::PhysicsRays { (const int32_t *)bufs[0], (const float *)bufs[1],
                                                         (const float *)bufs[2], (const float *)bufs[3] },
                              n, madrona_b200::PhysicsRayHits { (int32_t *)bufs[4], (float *)bufs[5],
                                                                (float *)bufs[6] });
        cudaDeviceSynchronize();      // the trace is enqueued on the executor's stream
        FILE *out = fopen(argv[3], "wb");
        if (!out) return 5;
        std::vector<unsigned char> tmp(n * 12);
        for (int k = 4; k < 7; k++) {
            cudaMemcpy(tmp.data(), bufs[k], bytes[k], 2 /* DtoH */);
            fwrite(tmp.data(), 1, bytes[k], out);
        }
        fclose(out);
        for (void *b : bufs) cudaFree(b);
    }
    cudaFree(dev_blob);
    printf("traced physics rays\n");
    return 0;
}
