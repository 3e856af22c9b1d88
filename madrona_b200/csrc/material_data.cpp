// material_data.cpp -- host-side material / texture upload: source materials and
// RGBA8 or BC7 pixels -> a render::MaterialData-compatible block (texture objects,
// their cudaArrays, madrona::Material array) for CudaBatchRenderConfig::materialData.
//
// Role of render::AssetProcessor::initMaterialData (src/render/asset_processor.cpp),
// with the same texture descriptor, so the ray caster samples textures made here
// and textures made by the reference the same way.  Unlike the reference, which
// aborts inside the CUDA calls, every input is checked first and a bad one is
// reported through mb2_last_error() without touching the GPU.
#include "../../include/madrona_b200.h"
#include "engine.hpp"
#include "render_bvh.h"

#include <algorithm>
#include <vector>

namespace mb2 {

struct MaterialBundle {
    int gpu = -1;
    std::vector<cudaTextureObject_t> texObjs;
    std::vector<cudaArray_t> arrays;       // == MaterialData::textureBuffers (host array)
    cudaTextureObject_t *dTextures = nullptr;
    RenderMaterial *dMaterials = nullptr;
    mb2_material_view view {};
};

static void destroyBundle(MaterialBundle *b)
{
    if (b->gpu >= 0) {
        cudaSetDevice(b->gpu);
        for (cudaTextureObject_t t : b->texObjs) cudaDestroyTextureObject(t);
        for (cudaArray_t a : b->arrays) cudaFreeArray(a);
        cudaFree(b->dTextures);
        cudaFree(b->dMaterials);
    }
    delete b;
}

static std::string validate(const mb2_source_material *materials, uint32_t num_materials,
                            const mb2_source_texture *textures, uint32_t num_textures, int gpu_id)
{
    if (gpu_id < 0) return "gpu_id must name a device (textures live on the GPU)";
    if (!materials || num_materials == 0) return "no materials";
    if (num_textures > 0 && !textures) return "num_textures > 0 but textures is NULL";
    for (uint32_t i = 0; i < num_textures; i++) {
        const mb2_source_texture &t = textures[i];
        const std::string at = "texture " + std::to_string(i) + ": ";
        if (t.format != 0 && t.format != 1) return at + "unknown format " + std::to_string(t.format);
        if (t.width == 0 || t.height == 0) return at + "zero width or height";
        if (!t.data) return at + "no pixel data";
        if (t.format == 1 && (t.width % 4 != 0 || t.height % 4 != 0)) {
            return at + "BC7 width and height must be multiples of 4";
        }
        // RGBA8: 4 bytes per texel; BC7: 16 bytes per 4 x 4 block, i.e. 1 byte per texel
        const uint64_t want = (uint64_t)t.width * t.height * (t.format == 0 ? 4u : 1u);
        if (t.num_bytes != want) {
            return at + "num_bytes is " + std::to_string(t.num_bytes) + ", " + std::to_string(t.width) + " x " +
                std::to_string(t.height) + (t.format == 0 ? " RGBA8" : " BC7") + " needs " + std::to_string(want);
        }
    }
    for (uint32_t i = 0; i < num_materials; i++) {
        const int32_t ti = materials[i].texture_idx;
        if (ti < -1 || ti >= (int64_t)num_textures) {
            return "material " + std::to_string(i) + ": texture_idx " + std::to_string(ti) + " is outside [-1, " +
                std::to_string(num_textures) + ")";
        }
    }
    return "";
}

}

using namespace mb2;

extern "C" {

mb2_material_data *mb2_init_material_data(const mb2_source_material *materials, uint32_t num_materials,
                                          const mb2_source_texture *textures, uint32_t num_textures,
                                          int gpu_id)
{
    const std::string bad = validate(materials, num_materials, textures, num_textures, gpu_id);
    if (!bad.empty()) {
        setError("mb2_init_material_data: " + bad);
        return nullptr;
    }
    MaterialBundle *b = new MaterialBundle();
    b->gpu = gpu_id;
    auto fail = [&](const char *what, cudaError_t e) {
        setError(std::string("mb2_init_material_data: ") + what + ": " + cudaGetErrorString(e));
        destroyBundle(b);
        return nullptr;
    };
    cudaError_t e = cudaSetDevice(gpu_id);
    if (e != cudaSuccess) return fail("cudaSetDevice", e);

    for (uint32_t i = 0; i < num_textures; i++) {
        const mb2_source_texture &t = textures[i];
        const bool bc7 = t.format == 1;
        const cudaChannelFormatDesc channel = bc7
            ? cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed7>()
            : cudaCreateChannelDesc<uchar4>();
        cudaArray_t arr = nullptr;
        if ((e = cudaMallocArray(&arr, &channel, t.width, t.height, cudaArrayDefault)) != cudaSuccess) {
            return fail("cudaMallocArray", e);
        }
        b->arrays.push_back(arr);
        // BC7: one row of 16-byte blocks covers 4 texel rows
        const size_t row_bytes = bc7 ? (size_t)16 * (t.width / 4) : (size_t)4 * t.width;
        const size_t rows = bc7 ? t.height / 4 : t.height;
        if ((e = cudaMemcpy2DToArray(arr, 0, 0, t.data, row_bytes, row_bytes, rows, cudaMemcpyHostToDevice)) !=
                cudaSuccess) {
            return fail("cudaMemcpy2DToArray", e);
        }
        cudaResourceDesc res = {};
        res.resType = cudaResourceTypeArray;
        res.res.array.array = arr;
        cudaTextureDesc desc = {};
        desc.addressMode[0] = cudaAddressModeWrap;
        desc.addressMode[1] = cudaAddressModeWrap;
        desc.filterMode = cudaFilterModeLinear;
        desc.readMode = cudaReadModeNormalizedFloat;
        desc.normalizedCoords = 1;
        cudaTextureObject_t obj = 0;
        if ((e = cudaCreateTextureObject(&obj, &res, &desc, nullptr)) != cudaSuccess) {
            return fail("cudaCreateTextureObject", e);
        }
        b->texObjs.push_back(obj);
    }

    std::vector<RenderMaterial> mats(num_materials);
    for (uint32_t i = 0; i < num_materials; i++) {
        for (int k = 0; k < 4; k++) mats[i].color[k] = materials[i].color[k];
        mats[i].textureIdx = materials[i].texture_idx;
        mats[i].roughness = materials[i].roughness;
        mats[i].metalness = materials[i].metalness;
    }
    // at least one entry each, so the device pointers are never NULL
    if ((e = cudaMalloc((void **)&b->dTextures, sizeof(cudaTextureObject_t) * std::max(num_textures, 1u))) !=
            cudaSuccess ||
        (e = cudaMalloc((void **)&b->dMaterials, sizeof(RenderMaterial) * num_materials)) != cudaSuccess) {
        return fail("cudaMalloc", e);
    }
    if ((num_textures > 0 &&
         (e = cudaMemcpy(b->dTextures, b->texObjs.data(), sizeof(cudaTextureObject_t) * num_textures,
                         cudaMemcpyHostToDevice)) != cudaSuccess) ||
        (e = cudaMemcpy(b->dMaterials, mats.data(), sizeof(RenderMaterial) * num_materials,
                        cudaMemcpyHostToDevice)) != cudaSuccess) {
        return fail("cudaMemcpy", e);
    }
    b->view.textures = b->dTextures;
    b->view.num_texture_buffers = num_textures;
    b->view.texture_buffers = b->arrays.empty() ? nullptr : (void *)b->arrays.data();
    b->view.materials = b->dMaterials;
    return (mb2_material_data *)b;
}

const mb2_material_view *mb2_material_data_view(const mb2_material_data *data)
{
    const MaterialBundle *b = (const MaterialBundle *)data;
    return b ? &b->view : nullptr;
}

void mb2_material_data_destroy(mb2_material_data *data)
{
    if (data) destroyBundle((MaterialBundle *)data);
}

}
