// render_state.h -- layouts shared by the NVRTC-side rendering API
// (device/madrona/render/ecs.hpp) and the ahead-of-time batch ray caster
// (kernels_render.cu).  SURVEY.md 8 rows a13-a15.
#pragma once

#include "mb2_state.h"
#include "render_bvh.h"

namespace mb2 {

struct RVec3 { float x, y, z; };
struct RQuat { float w, x, y, z; };

// == render::InstanceData (include/madrona/render/ecs.hpp:49-63) + the instance's
// world box (TLBVHNode in the reference)
struct RenderInstance {
    RVec3 position;
    RQuat rotation;
    RVec3 scale;
    i32 matID;            // MaterialOverride: -1 mesh default, -2 use `color`, else material index
    i32 objectID;
    u32 color;            // 0xRRGGBB (ColorOverride)
    float aabbMin[3];
    float aabbMax[3];
};

// == render::LightDesc (include/madrona/render/ecs.hpp:65-89), unpacked
struct RenderLight {
    u32 directional;      // LightDesc::Type: true = Directional, false = Spotlight
    u32 castShadow;
    RVec3 position;
    RVec3 direction;
    float cutoff;
    float intensity;
    u32 active;
};

constexpr int kMaxLightsPerWorld = 8;

// == render::PerspectiveCameraData (include/madrona/render/ecs.hpp:38-46)
struct RenderView {
    RVec3 position;
    RQuat rotation;       // inverse of the viewing entity's rotation
    float xScale;
    float yScale;
    float zNear;
    i32 worldIDX;
    i32 outputRow;        // row of the view's RaycastOutputArchetype entity
};

enum RenderCol : int { RCPosition = 0, RCRotation, RCScale, RCObjectID, RCRenderable, RCCount };

// == the LightDesc component as the simulator's compiler lays it out
struct LightDescComp {
    unsigned char type;       // enum Type : bool
    unsigned char castShadow;
    float position[3];
    float direction[3];
    float cutoff;
    float intensity;
    unsigned char active;
};
constexpr int kMaxRenderArchetypes = 16;

struct RenderArchetype {
    u32 archetype;
    i32 cols[RCCount];
    i32 colorCol;          // ColorOverride column or -1
    i32 matCol;            // MaterialOverride column or -1
};

struct ViewArchetype {
    u32 archetype;
    i32 posCol, rotCol, camCol;
};

struct RenderState {
    // ---- host config (before registerTypes)
    u32 enabled;
    u32 width, height;     // image size of every view: [height][width] pixels, row-major
    u32 rgbd;            // 1 = RGB + depth, 0 = depth only
    float nearPlane, farPlane;
    const MeshBVH *meshes;          // device, == CudaBatchRenderConfig::geoBVHData.meshBVHs
    u32 numMeshes;
    const RenderMaterial *materials;   // device, == materialData.materials (may be null)
    u32 debugHits;                  // MADRONA_B200_RENDER_DEBUG: keep (instance, triangle) per pixel

    // ---- written by the device-side RenderingSystem::registerTypes
    u32 registered;
    u32 cidRenderable, cidRenderCamera, cidColorOverride, cidMaterialOverride;
    u32 lightArchetype, cidLightDesc;
    u32 cidPosition, cidRotation, cidScale, cidObjectID;
    u32 outputArchetype;   // RaycastOutputArchetype
    u32 cidRGB, cidDepth;

    // ---- filled by the host after registerTypes
    u32 numRenderArchetypes;
    RenderArchetype renderables[kMaxRenderArchetypes];
    u32 numViewArchetypes;
    ViewArchetype viewers[kMaxRenderArchetypes];
    i32 rgbCol, depthCol;

    // Instances are one world-major list: world w's, in gather order, start at
    // instanceOffsets[w] (exclusive scan of instanceCounts).  The list, the TLAS nodes and
    // the large-world builder's scratch have one entry per row of the renderable tables
    // (instanceCapacity), mapped behind address ranges that grow with those tables.
    RenderInstance *instances;      // [instanceCapacity]
    i32 *instanceCounts;            // [numWorlds] visible renderables
    i32 *instanceOffsets;           // [numWorlds]
    i32 instanceCapacity;
    QBVHNode *tlasNodes;            // [instanceCapacity]; world w's tree at instanceOffsets[w], node 0 = root
    i32 *tlasNodeCounts;            // [numWorlds] (<= max(1, n - 1))
    i32 *tlasDepths;                // [numWorlds] levels of 4-wide nodes (0: no tree)
    unsigned long long *tlasKeys;   // [instanceCapacity] large-world builder: sorted Morton keys
    struct TLASBuildNode *tlasBuild;   // [instanceCapacity] large-world builder: binary / wide nodes
    i32 *largeWorlds;               // [numWorlds] worlds above the warp builder's size, world order
    u32 numLargeWorlds;
    u32 largeTicket;                // next entry of largeWorlds a builder block takes
    RenderLight *lights;            // [numWorlds][kMaxLightsPerWorld]
    i32 *lightCounts;               // [numWorlds]
    i32 lightCol;
    RenderView *views;              // [capacity of the output archetype]
    i32 maxViews;
    i32 *hitIDs;                    // debug: [maxViews][height*width][2] = (instance, triangle) or -1
    // exportCountsGPU (src/render/ecs_system.cpp:317-348): totals of the last prepare
    u32 totalNumViews;
    u32 totalNumInstances;

    // ---- host config: == materialData.textures / numTextureBuffers (device array of
    // cudaTextureObject_t; materials with textureIdx >= numTextures raise ErrRenderAsset)
    const unsigned long long *textures;
    u32 numTextures;
};

}
