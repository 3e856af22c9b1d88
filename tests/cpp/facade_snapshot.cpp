// madrona_b200::ExecutorSnapshot through the C++ facade (madrona_b200/host/madrona/mw_gpu.hpp):
// the cartpole fixture steps, saves, steps on, restores and steps again; the state after the
// second pass must equal the state after the first, byte for byte.
#include <madrona/mw_gpu.hpp>

#include <cstring>
#include <vector>

extern "C" int cudaMemcpy(void *, const void *, size_t, int);

struct Config { uint32_t maxSteps; };
struct WorldInit { uint32_t seed; };

int main(int argc, char **argv)
{
    const char *src = argc > 1 ? argv[1] : "sims/cartpole/sim.cpp";
    const uint32_t num_worlds = 64;
    Config cfg { 7 };   // short episodes: resets fall between the save and the restore
    std::vector<WorldInit> inits(num_worlds);
    for (uint32_t i = 0; i < num_worlds; i++) inits[i].seed = i;

    const char *sources[] = { src };
    const char *flags[] = { "-DCARTPOLE_FACADE_TEST=1" };

    madrona::MWCudaExecutor exec({
        .worldInitPtr = inits.data(),
        .numWorldInitBytes = sizeof(WorldInit),
        .userConfigPtr = &cfg,
        .numUserConfigBytes = sizeof(Config),
        .numWorldDataBytes = 0,
        .worldDataAlignment = 16,
        .numWorlds = num_worlds,
        .numTaskGraphs = 1,
        .numExportedBuffers = 5,
    }, {
        .userSources = madrona::Span<const char * const>(sources, 1),
        .userCompileFlags = madrona::Span<const char * const>(flags, 1),
    }, madrona::MWCudaExecutor::initCUDA(0));

    madrona::MWCudaLaunchGraph step = exec.buildLaunchGraphAllTaskGraphs();
    for (int i = 0; i < 3; i++) exec.run(step);

    std::vector<float> first(num_worlds * 4), second(num_worlds * 4), at_save(num_worlds * 4);
    cudaMemcpy(at_save.data(), exec.getExported(2), at_save.size() * sizeof(float), 2 /* DtoH */);
    {
        madrona_b200::ExecutorSnapshot snap = exec.snapshot();
        snap.save();
        for (int i = 0; i < 10; i++) exec.run(step);
        cudaMemcpy(first.data(), exec.getExported(2), first.size() * sizeof(float), 2);
        snap.restore();
        for (int i = 0; i < 10; i++) exec.run(step);
        cudaMemcpy(second.data(), exec.getExported(2), second.size() * sizeof(float), 2);
        if (memcmp(first.data(), second.data(), first.size() * sizeof(float)) != 0 ||
                memcmp(first.data(), at_save.data(), first.size() * sizeof(float)) == 0) {
            fprintf(stderr, "snapshot round trip differs\n");
            return 1;
        }
        printf("snapshot ok %lld bytes\n", (long long)snap.bytes());
    }
    return 0;
}
