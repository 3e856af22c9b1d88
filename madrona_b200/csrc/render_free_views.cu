// render_free_views.cu -- mb2_free_view records -> the ray caster's RenderView, on the device.
//
// A translation unit of its own because of its flags: kernels_render.cu is compiled with FMA
// contraction, this file (like the simulator's attachEntityToView, NVRTC --fmad=false) without.
// fovScale is computed here with attachEntityToView's expression, so a free view with a camera's
// pose and field of view gets that camera's bits, and with them the render graph's pixels.
#include "physics_host.hpp"
#include "render_state.h"

#include <madrona/math.hpp>

namespace mb2 {

// renderGatherViewsKernel's RenderView of a camera at `position` with the viewing entity's
// `rotation`: the conjugate rotation, xScale = fovScale, yScale = -fovScale
__global__ void __launch_bounds__(128)
renderConvertFreeViewsKernel(const mb2_free_view *in, RenderView *out, u32 n)
{
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const mb2_free_view f = in[i];
    const float fov_scale = 1.0f / tanf(madrona::math::toRadians(f.vfov_degrees * 0.5f));
    RenderView v;
    v.position = RVec3 { f.position[0], f.position[1], f.position[2] };
    v.rotation = RQuat { f.rotation[0], -f.rotation[1], -f.rotation[2], -f.rotation[3] };
    v.xScale = fov_scale;
    v.yScale = -fov_scale;
    v.zNear = 0.f;            // not used by the ray caster
    v.worldIDX = f.world;
    v.outputRow = (i32)i;
    out[i] = v;
}

void renderConvertFreeViews(const mb2_free_view *in, RenderView *out, uint32_t n, cudaStream_t s)
{
    renderConvertFreeViewsKernel<<<(n + 127) / 128, 128, 0, s>>>(in, out, n);
}

}
