"""Free views of the batch ray caster (mb2_render_free_views, MWCudaExecutor.renderFreeViews,
DESIGN 3.3): caller-given views of the last prepared scene into caller-owned buffers.

GPU: a free view with a gallery camera's pose, field of view, size and projection writes the
render graph's bytes for that camera (flat list, TLAS, large-world TLAS, textures; pinhole and
panorama; RGBD and depth-only executors); views of other sizes, fields of view and worlds in any
order against the float64 brute-force closest hit; no side effect on the exported columns;
snapshots; rejected calls launch nothing; the C++ facade against the Python call.  The block
split and the view conversion are modelled in tests/test_raycast_free_views_model.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from sims.render_assets import gallery_meshes
from test_raycast_free_views_model import build_facade
from test_render_aspect import _write_assets, camera_rays
from test_render_bvh import _closest_hits, _world_triangles
from test_render_panorama import panorama_rays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GALLERY_RGB, GALLERY_DEPTH, GALLERY_PROP_ENTITY, GALLERY_SEG, GALLERY_NORMALS = 8, 9, 10, 11, 12
OFFSET = np.array([0.0, 0.0, 0.25], dtype=np.float32)      # the gallery cameras' offset


def _visible(P):
    """prop rows of a gallery world that are drawn: the ground and all but every 17th prop"""
    return np.array([i for i in range(P) if i == 0 or i % 17 != 0], dtype=np.int64)


def _executor(name, W, width, height, rgbd=True, panorama=False, **cfg):
    from sims import make_executor
    return make_executor(name, W, rgbd=rgbd, segmentation=True, normals=True, panorama=panorama, seed=5,
                         width=width, height=height, **cfg)


def _col(ex, slot, dtype, shape):
    return ex.tensor(slot, dtype, shape).cpu().numpy().copy()


def _camera_views(ex, W, fov=70.0):
    """one free view per gallery camera, in output-row order (world w, camera v at 2 w + v)"""
    vpos, vrot = _col(ex, 6, "float32", (W, 2, 3)), _col(ex, 7, "float32", (W, 2, 4))
    return [(w, vpos[w, v] + OFFSET, vrot[w, v], fov) for w in range(W) for v in range(2)]


# ---- identity with the render graph -------------------------------------------------------------

CASES = {
    "flat_list_40_props": ("gallery", dict(num_props=40), [40] * 3),
    "tlas_100_props": ("gallery", dict(num_props=100), [100] * 3),
    # world 0: 142 visible props, past the warp builder's 128 (the large-world TLAS builder)
    "large_tlas_150_props": ("gallery_sized", dict(props=[150, 40]), [150, 40]),
    "textured_100_props": ("gallery_textured", dict(num_props=100), [100] * 2),
}
VIEWS = {"pinhole_64x32": (64, 32, False), "panorama_256x16": (256, 16, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("rgbd", [True, False], ids=["rgbd", "depth_only"])
@pytest.mark.parametrize("view", sorted(VIEWS))
@pytest.mark.parametrize("case", sorted(CASES))
def test_gpu_free_views_of_the_cameras_equal_the_render_graph_bytes(monkeypatch, case, view, rgbd):
    name, cfg, props = CASES[case]
    width, height, panorama = VIEWS[view]
    W = len(props)
    if name == "gallery_sized":
        monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", str(-(-sum(props) // W) + 64))
    ex = _executor(name, W, width, height, rgbd=rgbd, panorama=panorama, **cfg)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(3):
        ex.run(step)
    ex.run(render)
    want = dict(depth=_col(ex, GALLERY_DEPTH, "float32", (2 * W, height, width)),
                segmentation=_col(ex, GALLERY_SEG, "int32", (2 * W, height, width)),
                normals=_col(ex, GALLERY_NORMALS, "int8", (2 * W, height, width, 4)))
    if rgbd:
        want["rgb"] = _col(ex, GALLERY_RGB, "uint8", (2 * W, height, width, 4))
    got = ex.renderFreeViews(_camera_views(ex, W), width, height, panorama=panorama, rgb=rgbd, depth=True,
                             segmentation=True, normals=True)
    assert sorted(got) == sorted(want)
    for k in want:
        g = got[k].cpu().numpy()
        assert g.shape == want[k].shape and g.dtype == want[k].dtype, k
        assert np.array_equal(g.view(np.uint8), want[k].view(np.uint8)), (case, view, rgbd, k)
    assert (want["depth"] > 0).mean() > 0.2
    ex.close()


# ---- other sizes, fields of view and world orders against the brute-force closest hit ------------

SIZES = {"333x197": (333, 197), "1x1": (1, 1), "5x2": (5, 2), "1024x1024": (1024, 1024)}
# (world, camera, field of view) per view: one world several times, worlds out of order
LAYOUT = [(2, 0, 70.0), (0, 1, 50.0), (2, 1, 90.0), (1, 0, 70.0), (2, 0, 35.0), (0, 0, 120.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("panorama", [False, True], ids=["pinhole", "panorama"])
@pytest.mark.parametrize("size", sorted(SIZES))
def test_gpu_free_views_match_brute_force(size, panorama):
    width, height = SIZES[size]
    W, P = 3, 100
    ex = _executor("gallery", W, 40, 40, num_props=P)
    step = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(3):
        ex.run(step)
    rows = ex.exportedNumRows(0)
    pos, rot = _col(ex, 0, "float32", (rows, 3)), _col(ex, 1, "float32", (rows, 4))
    scale, obj = _col(ex, 2, "float32", (rows, 3)), _col(ex, 3, "int32", (rows,))
    entity = _col(ex, GALLERY_PROP_ENTITY, "int32", (rows, 2))[:, 1]
    vpos, vrot = _col(ex, 6, "float32", (W, 2, 3)), _col(ex, 7, "float32", (W, 2, 4))
    layout = LAYOUT[:1] if size == "1024x1024" else LAYOUT
    views = [(w, vpos[w, c] + OFFSET, vrot[w, c], fov) for w, c, fov in layout]
    got = ex.renderFreeViews(views, width, height, panorama=panorama, rgb=True, segmentation=True, normals=True)
    ex.close()
    depth, seg = got["depth"].cpu().numpy(), got["segmentation"].cpu().numpy()
    nrm, rgb = got["normals"].cpu().numpy(), got["rgb"].cpu().numpy()
    assert depth.shape == (len(views), height, width) and rgb.shape == (len(views), height, width, 4)
    # misses: seg == -1 and zero normals exactly where the depth is 0
    assert np.array_equal(seg == -1, depth == 0)
    assert np.array_equal((nrm == 0).all(axis=-1), depth == 0)
    assert (rgb[..., 3] == 255).all()
    meshes = gallery_meshes()
    rng = np.random.default_rng(7)
    checked = hits = total = 0
    for i, (w, pos_c, rot_c, fov) in enumerate(views):
        rows_w = w * P + _visible(P)
        tris, owner, _src = _world_triangles(meshes, pos[rows_w], rot[rows_w], scale[rows_w], obj[rows_w])
        cam = np.asarray(pos_c, dtype=np.float32).astype(np.float64)
        q = rot_c.astype(np.float64)
        fov_scale = 1.0 / np.tan(np.radians(fov / 2))
        rays = (panorama_rays if panorama else camera_rays)(cam, np.array([q[0], -q[1], -q[2], -q[3]]), fov_scale,
                                                            width, height)
        # at most 4096 pixels a view go to the float64 oracle
        pick = np.arange(len(rays)) if len(rays) <= 4096 else rng.choice(len(rays), 4096, replace=False)
        t, tri, t2 = _closest_hits(np.broadcast_to(cam, (len(pick), 3)), rays[pick], tris)
        d, s = depth[i].reshape(-1)[pick], seg[i].reshape(-1)[pick]
        want_hit, got_hit = np.isfinite(t), d > 0
        total += len(pick)
        # silhouettes may differ between the watertight fp32 test and float64 Moeller-Trumbore
        assert (want_hit != got_hit).sum() <= max(1, int(0.005 * len(pick))), (size, i)
        both = want_hit & got_hit
        hits += int(both.sum())
        np.testing.assert_allclose(d[both], t[both], rtol=1e-4, atol=1e-4)
        with np.errstate(invalid="ignore"):
            clear = both & ((t2 - t) > 1e-3 * np.maximum(t, 1.0))
        want_seg = entity[rows_w][owner[np.maximum(tri, 0)]]
        assert np.array_equal(s[clear], want_seg[clear]), (size, i)
        checked += int(clear.sum())
    if width * height > 16:
        assert hits > 0.2 * total and checked > 0.7 * hits


# ---- no side effects -----------------------------------------------------------------------------

def _exports(ex):
    """every exported column, the live rows' bytes"""
    out = {}
    for slot in range(13):
        n, b = ex.exportedNumRows(slot), ex.exportedRowBytes(slot)
        if n > 0 and b > 0:
            out[slot] = _col(ex, slot, "uint8", (n, b))
    return out


@pytest.mark.gpu
def test_gpu_free_views_leave_the_exported_columns_unchanged():
    W = 2
    runs = []
    for interleave in (False, True):
        ex = _executor("gallery", W, 48, 20, num_props=100)
        step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
        seen = []
        for _ in range(3):
            for g in (step, render):
                if interleave:
                    views = _camera_views(ex, W) + [(1, np.array([0.0, -6.0, 3.0]), np.array([1.0, 0, 0, 0]), 80.0)]
                    ex.renderFreeViews(views, 37, 11, rgb=True, segmentation=True, normals=True)
                    ex.renderFreeViews(views[:2], 64, 8, panorama=True, rgb=False, depth=True)
                ex.run(g)
                seen.append(_exports(ex))
        runs.append(seen)
        ex.close()
    for a, b in zip(*runs):
        assert sorted(a) == sorted(b)
        for slot in a:
            assert np.array_equal(a[slot], b[slot]), slot


# ---- snapshots -----------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_free_views_after_restore_equal_free_views_at_save():
    W = 2
    ex = _executor("gallery", W, 40, 40, num_props=100)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()

    def frame(views):
        got = ex.renderFreeViews(views, 96, 64, rgb=True, segmentation=True, normals=True)
        return {k: v.cpu().numpy() for k, v in got.items()}
    for _ in range(3):
        ex.run(step)
    ex.run(render)
    views = _camera_views(ex, W)
    with ex.snapshot() as snap:
        snap.save()
        at_save = frame(views)
        for _ in range(5):
            ex.run(step)
        # the props moved
        assert not np.array_equal(frame(views)["depth"], at_save["depth"])
        snap.restore()
        again = frame(views)
        for k in at_save:
            assert np.array_equal(again[k], at_save[k]), k
    ex.close()


# ---- rejected calls ------------------------------------------------------------------------------

def _call(ex, views, width, height, projection, outs):
    from madrona_b200.executor import _FreeViewC, _FreeViewOutputsC, _last_error
    arr = (_FreeViewC * max(len(views), 1))()
    for i, (w, p, r, f) in enumerate(views):
        arr[i] = _FreeViewC(w, (ctypes.c_float * 3)(*p), (ctypes.c_float * 4)(*r), f)
    ptrs = _FreeViewOutputsC(*[None if t is None else t.data_ptr() for t in outs])
    rc = ex._lib.mb2_render_free_views(ex._h, arr, len(views), width, height, projection, ctypes.byref(ptrs), None)
    return rc, _last_error(ex._lib)


GOOD = (0, (0.0, -5.0, 2.0), (1.0, 0.0, 0.0, 0.0), 70.0)
INVALID = [
    ("no_views", [], 8, 8, 0, "num_views is 0"),
    ("world_past_the_end", [GOOD, (2, GOOD[1], GOOD[2], 70.0)], 8, 8, 0, r"view 1: world 2 is outside \[0, 2\)"),
    ("negative_world", [(-1, GOOD[1], GOOD[2], 70.0)], 8, 8, 0, r"view 0: world -1 is outside \[0, 2\)"),
    ("nan_position", [(0, (0.0, float("nan"), 2.0), GOOD[2], 70.0)], 8, 8, 0, "view 0: position, rotation or "
     "vfov_degrees is not finite"),
    ("inf_rotation", [(0, GOOD[1], (1.0, float("inf"), 0.0, 0.0), 70.0)], 8, 8, 0, "is not finite"),
    ("nan_fov", [(0, GOOD[1], GOOD[2], float("nan"))], 8, 8, 0, "is not finite"),
    ("zero_fov", [(0, GOOD[1], GOOD[2], 0.0)], 8, 8, 0, r"vfov_degrees = 0.000000 is outside \(0, 180\)"),
    ("fov_180", [(0, GOOD[1], GOOD[2], 180.0)], 8, 8, 0, r"is outside \(0, 180\)"),
    ("zero_width", [GOOD], 0, 8, 0, "width and height must be at least 1"),
    ("zero_height", [GOOD], 8, 0, 0, "width and height must be at least 1"),
    ("image_past_32_bits", [GOOD], 65536, 16384, 0, "exceed the 32-bit component size"),
    ("projection_2", [GOOD], 8, 8, 2, r"projection = 2 is not 0 \(pinhole\) or 1 \(panorama\)"),
]


@pytest.mark.gpu
def test_gpu_rejected_free_views_launch_nothing():
    import torch
    import madrona_b200 as mb
    ex = _executor("gallery", 2, 40, 40, num_props=40)
    ex.run(ex.buildLaunchGraphAllTaskGraphs())
    dev = f"cuda:{ex.gpu_id}"
    bufs = [torch.full((4, 8, 8, 4), 0x5A, dtype=torch.uint8, device=dev) for _ in range(4)]
    for _name, views, width, height, projection, message in INVALID:
        rc, err = _call(ex, views, width, height, projection, bufs)
        assert rc == 1 and err.startswith("mb2_render_free_views: "), (_name, err)
        assert __import__("re").search(message, err), (_name, err)
    rc, err = _call(ex, [GOOD], 8, 8, 0, [None] * 4)
    assert rc == 1 and "every output (rgb, depth, segmentation, normals) is NULL" in err
    torch.cuda.synchronize()
    assert all((b == 0x5A).all() for b in bufs)
    with pytest.raises(mb.MadronaB200Error, match="vfov_degrees"):
        ex.renderFreeViews([(0, GOOD[1], GOOD[2], 200.0)], 8, 8)
    # the device is healthy: a valid call renders
    got = ex.renderFreeViews(_camera_views(ex, 2), 40, 40)
    torch.cuda.synchronize()
    assert (got["depth"] > 0).float().mean().item() > 0.3
    ex.close()
    # an executor without a renderer
    from sims import make_executor
    ex = make_executor("cartpole", 2)
    rc, err = _call(ex, [GOOD], 8, 8, 0, bufs)
    assert rc == 1 and "the executor has no renderer" in err
    torch.cuda.synchronize()
    assert all((b == 0x5A).all() for b in bufs)
    ex.close()


# ---- asynchronous calls --------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_free_views_on_a_caller_stream_equal_the_synchronous_call():
    import torch
    W = 2
    ex = _executor("gallery", W, 40, 40, num_props=40)
    ex.run(ex.buildLaunchGraphAllTaskGraphs())
    views = _camera_views(ex, W)
    want = ex.renderFreeViews(views, 50, 30, segmentation=True)
    # a structured array works as well as tuples
    arr = np.zeros(len(views), dtype=[("world", "<i4"), ("position", "<f4", 3), ("rotation", "<f4", 4),
                                      ("vfov_degrees", "<f4")])
    for i, v in enumerate(views):
        arr[i] = v
    s = torch.cuda.Stream()
    # ordered after the executor's stream (the steps), as the ordering rule asks
    s.wait_stream(torch.cuda.ExternalStream(ex.stream))
    got = ex.renderFreeViews(arr, 50, 30, segmentation=True, stream=s)
    s.synchronize()
    for k in want:
        assert torch.equal(got[k], want[k]), k
    ex.close()


# ---- the C++ facade ------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_facade_free_views_match_python_call(tmp_path):
    from sims import make_executor
    exe = build_facade(tmp_path)
    assets, out = str(tmp_path / "assets.bin"), str(tmp_path / "frame.bin")
    _write_assets(assets)
    res = subprocess.run([exe, os.path.join(ROOT, "sims", "gallery", "sim.cpp"), assets, out],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    raw = np.fromfile(out, dtype=np.uint8)
    n = 3 * 40 * 24 * 4
    assert raw.size == 4 * n
    W = 2
    ex = make_executor("gallery", W, num_props=40, seed=5, rgbd=True, segmentation=True, normals=True,
                       width=64, height=32)
    step = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(3):
        ex.run(step)
    vpos, vrot = _col(ex, 6, "float32", (W, 2, 3)), _col(ex, 7, "float32", (W, 2, 4))
    views = [(w, vpos[w, c] + OFFSET, vrot[w, c], 60.0) for w, c in [(1, 0), (0, 1), (1, 1)]]
    want = ex.renderFreeViews(views, 40, 24, rgb=True, segmentation=True, normals=True)
    ex.close()
    for i, k in enumerate(["rgb", "depth", "segmentation", "normals"]):
        assert np.array_equal(raw[i * n:(i + 1) * n], want[k].cpu().numpy().reshape(-1).view(np.uint8)), k
    assert (want["depth"] > 0).float().mean().item() > 0.3
