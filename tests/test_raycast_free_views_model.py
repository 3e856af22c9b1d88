"""Free views of the batch ray caster (mb2_render_free_views, DESIGN 3.3), without a GPU.

- The block split of renderRaycastKernel: block x of a view takes tiles x * warps + warp,
  stepping by gridDim.x * warps.  Every pixel of every view is traced exactly once for any
  gridDim.x, and gridDim.x = 1 (the render graph) keeps the tile order of one block per view.
- The free path's grid: the chunk count renderFreeViews picks from the view count and size.
- The conversion of a free view into the ray caster's RenderView, against the gather kernel's
  formulas: the pinhole rays of the converted view are the camera's rays.
- The C ABI's structs against the ctypes ones, a null executor's rejection, and the C++
  facade's renderFreeViews against the stand-alone and the reference headers.
The GPU side is tests/test_render_free_views.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from test_render_aspect import camera_rays
from test_render_bvh import _quat_rotate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WARPS = 256 // 32             # warps of a ray-caster block
MIN_BLOCKS = 3                # kRaycastMinBlocks
H100_SMS = 132


# ---- the block split -----------------------------------------------------------------------------

def tiling(width, height):
    """the kernel's tiles: 8 x 4 pixels, 32 x 1 for images under 4 rows -> (tile_w, tile_h, tiles_x, tiles)"""
    tile_shift = 5 if height < 4 else 3
    tile_w, tile_h = 1 << tile_shift, 32 >> tile_shift
    tiles_x = (width + tile_w - 1) >> tile_shift
    return tile_w, tile_h, tiles_x, tiles_x * ((height + tile_h - 1) // tile_h)


def warp_pixels(width, height, grid_x, block_x, warp):
    """the (px, py) a warp of block x traces, in order (lanes of a tile, then its next tile)"""
    tile_w, tile_h, tiles_x, tiles = tiling(width, height)
    out = []
    tile = block_x * WARPS + warp
    while tile < tiles:
        tx0, ty0 = (tile % tiles_x) * tile_w, (tile // tiles_x) * tile_h
        for lane in range(32):
            px, py = tx0 + (lane & (tile_w - 1)), ty0 + lane // tile_w
            if px < width and py < height:
                out.append((px, py))
        tile += grid_x * WARPS
    return out


def parent_warp_pixels(width, height, warp):
    """one block per view, as the render graph always ran: tile = warp, stepping by the warps"""
    tile_w, tile_h, tiles_x, tiles = tiling(width, height)
    out = []
    for tile in range(warp, tiles, WARPS):
        tx0, ty0 = (tile % tiles_x) * tile_w, (tile // tiles_x) * tile_h
        for lane in range(32):
            px, py = tx0 + (lane & (tile_w - 1)), ty0 + lane // tile_w
            if px < width and py < height:
                out.append((px, py))
    return out


SPLIT_SIZES = [(1, 1), (7, 3), (8, 4), (33, 5), (64, 64), (1920, 1080)]


@pytest.mark.parametrize("size", SPLIT_SIZES, ids=[f"{w}x{h}" for w, h in SPLIT_SIZES])
def test_block_split_traces_every_pixel_exactly_once(size):
    width, height = size
    tiles = tiling(width, height)[3]
    for grid_x in sorted({1, 3, tiles // WARPS + 2, tiles + 5}):
        count = np.zeros((height, width), dtype=np.int64)
        for bx in range(grid_x):
            for warp in range(WARPS):
                px = warp_pixels(width, height, grid_x, bx, warp)
                if px:
                    xs, ys = np.array(px).T
                    np.add.at(count, (ys, xs), 1)
        assert (count == 1).all(), (size, grid_x)


@pytest.mark.parametrize("size", SPLIT_SIZES[:5], ids=[f"{w}x{h}" for w, h in SPLIT_SIZES[:5]])
def test_one_block_per_view_keeps_the_tile_order(size):
    width, height = size
    for warp in range(WARPS):
        assert warp_pixels(width, height, 1, 0, warp) == parent_warp_pixels(width, height, warp)


def test_images_under_four_rows_keep_every_lane_on_a_pixel():
    assert tiling(7, 3)[:2] == (32, 1)
    assert tiling(8, 4)[:2] == (8, 4)


def free_grid(n, width, height, sms=H100_SMS):
    """renderFreeViews' grid: (tile chunks per view = gridDim.x, view blocks = gridDim.y)"""
    tiles = tiling(width, height)[3]
    resident = sms * MIN_BLOCKS * 8
    chunks = max(1, min(-(-resident // n), -(-tiles // WARPS)))
    return chunks, max(1, min(n, resident // chunks))


def test_free_grid_fills_the_gpu_with_few_large_views():
    # one 1920 x 1080 view: the 8 rounds of resident blocks of the render graph, all on it
    assert free_grid(1, 1920, 1080) == (3168, 1)
    # 8 views of 512 x 512: 396 chunks each
    assert free_grid(8, 512, 512) == (396, 8)
    # 4096 views of 64 x 64: one block per view, as the render graph launches
    assert free_grid(4096, 64, 64) == (1, 3168)
    # a chunk has a tile for every warp; tiny images get one chunk
    for n, w, h in [(1, 1, 1), (3, 5, 2), (1, 64, 64), (2, 333, 197), (1, 1024, 1024)]:
        chunks, blocks = free_grid(n, w, h)
        assert 1 <= chunks <= max(1, -(-tiling(w, h)[3] // WARPS))
        assert 1 <= blocks <= min(n, 65535)
    assert free_grid(1, 1, 1) == (1, 1)


# ---- free view -> RenderView ------------------------------------------------------------------------

def convert(view):
    """render_free_views.cu in float32: the conjugate rotation, xScale = fovScale,
    yScale = -fovScale, fovScale = 1 / tanf(toRadians(vfov * 0.5))"""
    f32 = np.float32
    _world, pos, rot, vfov = view
    fov_scale = f32(1.0) / f32(np.tan(f32(f32(np.pi) / f32(180.0)) * (f32(vfov) * f32(0.5))))
    q = np.asarray(rot, dtype=f32)
    return dict(position=np.asarray(pos, dtype=f32), rotation=np.array([q[0], -q[1], -q[2], -q[3]], dtype=f32),
                xScale=fov_scale, yScale=-fov_scale)


def kernel_pinhole_rays(rv, width, height):
    """renderRaycastKernel's pinhole rays of a RenderView, in float64"""
    q_inv = rv["rotation"].astype(np.float64)
    q = np.array([q_inv[0], -q_inv[1], -q_inv[2], -q_inv[3]])      # rot.inv()
    fwd = _quat_rotate(q, np.array([0.0, 1.0, 0.0]))
    fwd /= np.linalg.norm(fwd)
    u = _quat_rotate(q, np.array([1.0, 0.0, 0.0]))
    vv = np.cross(fwd, u)
    vv /= np.linalg.norm(vv)
    h = 1.0 / (-float(rv["yScale"]))
    horizontal, vertical = u * 2 * h * (width / height), vv * 2 * h
    pos = rv["position"].astype(np.float64)
    ll = pos - horizontal / 2 - vertical / 2 + fwd
    pu = (np.arange(width) + 0.5) / width
    pv = (np.arange(height) + 0.5) / height
    d = ll[None, None] + pu[None, :, None] * horizontal + pv[:, None, None] * vertical - pos
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return d.reshape(-1, 3)


def test_converted_view_has_the_gather_kernels_frame_and_scales():
    rng = np.random.default_rng(3)
    for _ in range(20):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        pos = rng.normal(size=3) * 5
        vfov = rng.uniform(10, 170)
        rv = convert((0, pos, q, vfov))
        # renderGatherViewsKernel: v.rotation = q.inv(), xScale = fovScale, yScale = -fovScale
        assert np.array_equal(rv["rotation"], np.array([q[0], -q[1], -q[2], -q[3]], dtype=np.float32))
        assert rv["xScale"] == -rv["yScale"] > 0
        np.testing.assert_allclose(float(rv["xScale"]), 1.0 / np.tan(np.radians(vfov / 2)), rtol=1e-5)
        # the rays of the converted view are the camera's (tests/test_render_aspect.py's model)
        want = camera_rays(pos.astype(np.float32).astype(np.float64), rv["rotation"].astype(np.float64),
                           float(rv["xScale"]), 24, 10)
        np.testing.assert_allclose(kernel_pinhole_rays(rv, 24, 10), want, atol=1e-12)
        # the camera looks along the rotated +y axis, +x to its right
        fwd = _quat_rotate(q, np.array([0.0, 1.0, 0.0]))
        assert np.dot(kernel_pinhole_rays(rv, 1, 1)[0], fwd) > 1 - 1e-6


def test_gallery_camera_fov_scale():
    """70 degrees, the gallery's cameras: the scale the render tests' float64 rays use"""
    rv = convert((0, np.zeros(3), np.array([1.0, 0, 0, 0]), 70.0))
    np.testing.assert_allclose(float(rv["xScale"]), 1.0 / np.tan(np.radians(35.0)), rtol=1e-6)


# ---- the C ABI and the C++ facade (no GPU needed) -------------------------------------------------

def test_free_view_structs_match_the_c_header(tmp_path):
    from madrona_b200.executor import _FreeViewC, _FreeViewOutputsC
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "madrona_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(mb2_free_view), '
                   'offsetof(mb2_free_view, world), offsetof(mb2_free_view, position), '
                   'offsetof(mb2_free_view, rotation), offsetof(mb2_free_view, vfov_degrees), '
                   'sizeof(mb2_free_view_outputs), offsetof(mb2_free_view_outputs, depth), '
                   'offsetof(mb2_free_view_outputs, segmentation), offsetof(mb2_free_view_outputs, normals));'
                   ' return 0; }\n')
    exe = str(tmp_path / "layout")
    res = subprocess.run(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    want = [ctypes.sizeof(_FreeViewC), _FreeViewC.world.offset, _FreeViewC.position.offset,
            _FreeViewC.rotation.offset, _FreeViewC.vfov_degrees.offset, ctypes.sizeof(_FreeViewOutputsC),
            _FreeViewOutputsC.depth.offset, _FreeViewOutputsC.segmentation.offset, _FreeViewOutputsC.normals.offset]
    assert got == want
    assert got[0] == 36
    # the numpy record the Python binding builds is the same layout
    assert np.dtype(_FreeViewC).itemsize == 36


def test_null_executor_or_views_are_rejected():
    import madrona_b200 as mb
    from madrona_b200.executor import _FreeViewC, _FreeViewOutputsC, _last_error
    lib = mb.load_library()
    outs = _FreeViewOutputsC(None, 1, None, None)
    views = (_FreeViewC * 1)()
    assert lib.mb2_render_free_views(None, views, 1, 8, 8, 0, ctypes.byref(outs), None) == 1
    assert "mb2_render_free_views: null executor or views" in _last_error(lib)


def build_facade(tmp_path):
    exe = str(tmp_path / "facade_render_free_views")
    cmd = ["g++", "-std=c++20", "-O1", "-I" + os.path.join(ROOT, "madrona_b200", "host"),
           os.path.join(ROOT, "tests", "cpp", "facade_render_free_views.cpp"), "-o", exe,
           "-L" + os.path.join(ROOT, "madrona_b200"), "-lmadrona_b200",
           "-Wl,-rpath," + os.path.join(ROOT, "madrona_b200"),
           "-L/usr/local/cuda/lib64", "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    return exe


def test_facade_render_free_views_compiles(tmp_path):
    build_facade(tmp_path)


REF_INCLUDE = "/root/reference/include"


@pytest.mark.skipif(not os.path.isdir(REF_INCLUDE), reason="reference headers not on this box")
def test_facade_render_free_views_compiles_against_reference_headers(tmp_path):
    # the reference's Span (madrona/span.hpp) in renderFreeViews' signature
    src = tmp_path / "mgr.cpp"
    src.write_text('#include <madrona/span.hpp>\n#include <madrona/mw_gpu.hpp>\n'
                   'void render(madrona::MWCudaExecutor &exec, const madrona_b200::FreeView *views, int n,\n'
                   '            void *depth) {\n'
                   '    exec.renderFreeViews(madrona::Span<const madrona_b200::FreeView>(views, n),\n'
                   '                         madrona_b200::RenderImageSize { 64, 48 },\n'
                   '                         madrona_b200::RenderProjection::Panorama,\n'
                   '                         madrona_b200::FreeViewOutputs { nullptr, depth, nullptr, nullptr });\n'
                   '}\n')
    cmd = ["g++", "-std=c++20", "-O1", "-w", "-D_LIBCPP_VERSION=190000", "-c",
           "-include", os.path.join(ROOT, "tests", "cpp", "ref_shim.h"),
           "-I" + os.path.join(ROOT, "madrona_b200", "host"), "-I" + REF_INCLUDE, "-I/usr/local/cuda/include",
           str(src), "-o", str(tmp_path / "mgr.o")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
