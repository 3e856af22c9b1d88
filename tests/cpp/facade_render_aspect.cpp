// A Manager-style snippet that asks the C++ facade (madrona_b200/host/madrona/mw_gpu.hpp) for
// non-square images through the MWCudaExecutor overload with a madrona_b200::RenderImageSize.
// It builds the gallery fixture's render assets through the C ABI, steps the gallery 3 times,
// renders one 64 x 32 RGBD frame and writes the RGB and depth exports to a file:
//   facade_render_aspect <gallery sim.cpp> <assets file> <output file>
// The assets file (written by tests/test_render_aspect.py) holds, little-endian:
//   u32 meshes; per mesh u32 vertices, u32 triangles, i32 material, f32 xyz[], u32 indices[];
//   u32 materials; per material f32 color[4], i32 texture, f32 roughness, f32 metalness.
#include <madrona/mw_gpu.hpp>

#include <cstdio>
#include <string>
#include <vector>

extern "C" int cudaMemcpy(void *, const void *, size_t, int);

struct Config { uint32_t numProps; uint32_t numLights; };
struct WorldInit { uint32_t seed; };

static bool readAll(FILE *f, void *dst, size_t bytes) { return fread(dst, 1, bytes, f) == bytes; }

int main(int argc, char **argv)
{
    if (argc < 4) return 2;
    constexpr uint32_t num_worlds = 2, width = 64, height = 32;

    FILE *f = fopen(argv[2], "rb");
    if (!f) return 3;
    uint32_t num_meshes = 0;
    readAll(f, &num_meshes, 4);
    std::vector<std::vector<float>> positions(num_meshes);
    std::vector<std::vector<uint32_t>> indices(num_meshes);
    std::vector<mb2_mesh_source> meshes(num_meshes);
    for (uint32_t m = 0; m < num_meshes; m++) {
        uint32_t nv = 0, nt = 0;
        int32_t mat = -1;
        readAll(f, &nv, 4);
        readAll(f, &nt, 4);
        readAll(f, &mat, 4);
        positions[m].resize(3 * nv);
        indices[m].resize(3 * nt);
        if (!readAll(f, positions[m].data(), 12 * nv) || !readAll(f, indices[m].data(), 12 * nt)) return 3;
        meshes[m] = mb2_mesh_source { positions[m].data(), nullptr, nv, indices[m].data(), nt, mat };
    }
    uint32_t num_materials = 0;
    readAll(f, &num_materials, 4);
    std::vector<mb2_source_material> materials(num_materials);
    if (!readAll(f, materials.data(), sizeof(mb2_source_material) * num_materials)) return 3;
    fclose(f);

    CUcontext ctx = madrona::MWCudaExecutor::initCUDA(0);
    mb2_mesh_bvh_data *bvh = mb2_build_mesh_bvhs(meshes.data(), num_meshes, 0);
    mb2_material_data *mats = mb2_init_material_data(materials.data(), num_materials, nullptr, 0, 0);
    if (!bvh || !mats) {
        fprintf(stderr, "madrona_b200: assets: %s\n", mb2_last_error());
        return 4;
    }
    const mb2_material_view *mv = mb2_material_data_view(mats);

    madrona::CudaBatchRenderConfig render_cfg {};
    render_cfg.renderMode = madrona::CudaBatchRenderConfig::RenderMode::RGBD;
    memcpy(&render_cfg.geoBVHData, mb2_mesh_bvh_data_view(bvh, 1), sizeof(render_cfg.geoBVHData));
    render_cfg.materialData.textures = mv->textures;
    render_cfg.materialData.numTextureBuffers = mv->num_texture_buffers;
    render_cfg.materialData.textureBuffers = mv->texture_buffers;
    render_cfg.materialData.materials = mv->materials;
    render_cfg.renderResolution = 0;
    render_cfg.nearPlane = 0.001f;
    render_cfg.farPlane = 1000.f;

    Config cfg { 40, 5 };
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
            .numExportedBuffers = 10,
        }, {
            .userSources = madrona::Span<const char * const>(sources, 1),
            .userCompileFlags = madrona::Span<const char * const>(flags, 1),
        }, ctx, render_cfg, madrona_b200::RenderImageSize { width, height });

        madrona::MWCudaLaunchGraph step = exec.buildLaunchGraphAllTaskGraphs();
        madrona::MWCudaLaunchGraph render = exec.buildRenderGraph();
        for (int i = 0; i < 3; i++) exec.run(step);
        exec.run(render);

        const size_t bytes = (size_t)2 * num_worlds * width * height * 4;
        std::vector<unsigned char> rgb(bytes), depth(bytes);
        cudaMemcpy(rgb.data(), exec.getExported(8), bytes, 2 /* DtoH */);
        cudaMemcpy(depth.data(), exec.getExported(9), bytes, 2 /* DtoH */);
        FILE *out = fopen(argv[3], "wb");
        if (!out) return 5;
        fwrite(rgb.data(), 1, bytes, out);
        fwrite(depth.data(), 1, bytes, out);
        fclose(out);
    }
    mb2_material_data_destroy(mats);
    mb2_mesh_bvh_data_destroy(bvh);
    printf("rendered %u x %u\n", width, height);
    return 0;
}
