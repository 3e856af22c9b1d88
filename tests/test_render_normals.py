"""Surface normal output of the batch ray caster (mb2_render_config::normals, DESIGN 3.3): every
view gets a row-major [H][W] image of int8 x, y, z, w, round(127 n) of the unit geometric
normal of the triangle the pixel's primary ray hits first, in the view's frame (x = n.u,
y = n.vv, z = n.forward), turned to face the camera, w = 0; all zero where the ray hits nothing.

GPU: every hit pixel against the float64 normal of the triangle the debug hit buffer names
(its world-space edges, tests/test_render_bvh.py's transform), oriented by the float64 pixel
ray, on the flat list (40 props), the TLAS (100 props) and the large-world TLAS builder (a world
of 150 props), with a square and a non-square pinhole and a panorama; misses exactly where the
depth is 0; RGB, depth and segmentation byte-identical with the output on and off; snapshots;
the C++ facade's RenderOutputs against the Python-created executor.  The float32 normal is
modelled in tests/test_raycast_normals_model.py."""
import os
import subprocess

import numpy as np
import pytest

from sims.render_assets import gallery_meshes
from test_raycast_normals_model import build_facade
from test_render_aspect import FOV_SCALE, _write_assets, camera_rays
from test_render_bvh import _quat_rotate, _world_triangles
from test_render_panorama import panorama_rays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GALLERY_RGB, GALLERY_DEPTH, GALLERY_SEG, GALLERY_NORMALS = 8, 9, 11, 12


def _visible(P):
    """prop rows of a gallery world that are drawn: the ground and all but every 17th prop"""
    return np.array([i for i in range(P) if i == 0 or i % 17 != 0], dtype=np.int64)


def _render(name, W, width, height, steps=3, rgbd=True, normals=True, panorama=False, **cfg):
    """`steps` steps of a gallery fixture (the props spin and bob), then one frame with
    segmentation; flat exported columns (rows of all worlds)"""
    from sims import make_executor
    ex = make_executor(name, W, rgbd=rgbd, segmentation=True, normals=normals, panorama=panorama, seed=5,
                       width=width, height=height, **cfg)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(steps):
        ex.run(step)
    ex.run(render)
    rows = ex.exportedNumRows(0)

    def col(slot, dtype, shape):
        return ex.tensor(slot, dtype, shape).cpu().numpy().copy()
    out = dict(rows=rows, depth=col(GALLERY_DEPTH, "float32", (2 * W, height, width)),
               seg=col(GALLERY_SEG, "int32", (2 * W, height, width)),
               normal_row_bytes=ex.exportedRowBytes(GALLERY_NORMALS),
               pos=col(0, "float32", (rows, 3)), rot=col(1, "float32", (rows, 4)),
               scale=col(2, "float32", (rows, 3)), obj=col(3, "int32", (rows,)),
               vpos=col(6, "float32", (W, 2, 3)), vrot=col(7, "float32", (W, 2, 4)))
    if rgbd:
        out["rgb"] = col(GALLERY_RGB, "uint8", (2 * W, height, width, 4))
    if normals:
        out["normals"] = col(GALLERY_NORMALS, "int8", (2 * W, height, width, 4))
    if os.environ.get("MADRONA_B200_RENDER_DEBUG") == "1":
        out["hits"] = ex.renderDebugHits(2 * W, height, width).cpu().numpy()
    ex.close()
    return out


def view_frame(vrot):
    """the kernel's view frame in float64 (u, vv, forward), from the exported view rotation"""
    q = vrot.astype(np.float64)
    fwd = _quat_rotate(q, np.array([0.0, 1.0, 0.0]))
    fwd /= np.linalg.norm(fwd)
    u = _quat_rotate(q, np.array([1.0, 0.0, 0.0]))
    vv = np.cross(fwd, u)
    vv /= np.linalg.norm(vv)
    return u, vv, fwd


# ---- every hit pixel against the float64 normal of the debug buffer's triangle ---------------------

CASES = {
    "flat_list_40_props": ("gallery", dict(num_props=40), [40] * 3),
    "tlas_100_props": ("gallery", dict(num_props=100), [100] * 3),
    # world 0: 142 visible props, past the warp builder's 128 (the large-world TLAS builder);
    # world 1 on the flat list
    "large_tlas_150_props": ("gallery_sized", dict(props=[150, 40]), [150, 40]),
}
VIEWS = {
    "pinhole_40x40": (40, 40, False),
    "pinhole_64x32": (64, 32, False),
    "panorama_256x16": (256, 16, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("view", sorted(VIEWS))
@pytest.mark.parametrize("case", sorted(CASES))
def test_gpu_normals_match_the_float64_normal_of_the_hit_triangle(monkeypatch, case, view):
    import madrona_b200 as mb
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    name, cfg, props = CASES[case]
    width, height, panorama = VIEWS[view]
    W = len(props)
    if name == "gallery_sized":
        # tables with room for every prop from the start (tests/test_render_large_worlds.py)
        monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", str(-(-sum(props) // W) + 64))
    r = _render(name, W, width, height, panorama=panorama, **cfg)
    assert r["rows"] == sum(props)
    assert r["normal_row_bytes"] == width * height * 4
    meshes = gallery_meshes()
    src_of = mb.MeshBVHData(meshes, gpu_id=-1).triangle_sources()
    first_tri = np.cumsum([0] + [len(m[1]) for m in meshes])
    starts = np.concatenate([[0], np.cumsum(props)[:-1]])
    hit_total = grazing = 0
    for w in range(W):
        rows = starts[w] + _visible(props[w])
        obj_w = r["obj"][rows]
        tris, _owner, _src = _world_triangles(meshes, r["pos"][rows], r["rot"][rows], r["scale"][rows], obj_w)
        # first world triangle of every instance (_world_triangles keeps source order)
        inst_start = np.concatenate([[0], np.cumsum([len(meshes[o][1]) for o in obj_w])[:-1]])
        for v in range(2):
            view_i = 2 * w + v
            cam = r["vpos"][w, v].astype(np.float64) + np.array([0.0, 0.0, 0.25])
            q = r["vrot"][w, v].astype(np.float64)
            q_inv = np.array([q[0], -q[1], -q[2], -q[3]])
            rays = (panorama_rays if panorama else camera_rays)(cam, q_inv, FOV_SCALE, width, height)
            u, vv, fwd = view_frame(q)
            got = r["normals"][view_i].reshape(-1, 4).astype(np.int64)
            depth = r["depth"][view_i].reshape(-1)
            inst, tri = r["hits"][view_i].reshape(-1, 2)[:, 0], r["hits"][view_i].reshape(-1, 2)[:, 1]
            hit = inst >= 0
            # misses: all zero exactly where the depth is 0; w is always 0
            assert np.array_equal((got == 0).all(axis=1), depth == 0), (case, view, w, v)
            assert np.array_equal(hit, depth > 0)
            assert (got[:, 3] == 0).all()
            # the triangle the debug buffer names, in float64
            k = np.nonzero(hit)[0]
            src = src_of[first_tri[obj_w[inst[k]]] + tri[k]]
            t = tris[inst_start[inst[k]] + src]
            n = np.cross(t[:, 1] - t[:, 0], t[:, 2] - t[:, 0])
            n /= np.linalg.norm(n, axis=1, keepdims=True)
            cos = (n * rays[k]).sum(1)
            n = np.where(cos[:, None] > 0, -n, n)
            want = np.clip(np.rint(127 * np.stack([n @ u, n @ vv, n @ fwd], axis=1)), -127, 127).astype(np.int64)
            g = got[k, :3]
            ok = np.abs(g - want).max(axis=1) <= 1
            # where the ray grazes the surface the orientation is not resolved: either sign
            graze = np.abs(cos) < 1e-4
            ok |= graze & (np.abs(g + want).max(axis=1) <= 1)
            assert ok.all(), (case, view, w, v, g[~ok][:5], want[~ok][:5], cos[~ok][:5])
            hit_total += len(k)
            grazing += int(graze.sum())
    assert hit_total > 0.25 * 2 * W * width * height
    assert grazing < 0.01 * hit_total


# ---- the other outputs do not change -----------------------------------------------------------------

SIZES = {"pinhole_64x32": (64, 32, False), "panorama_128x8": (128, 8, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("view", sorted(SIZES))
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_props", "flat_list_40_props"])
def test_gpu_rgb_depth_and_segmentation_are_byte_identical_with_normals_on_and_off(P, view):
    width, height, panorama = SIZES[view]
    for rgbd in (True, False):
        off = _render("gallery", 2, width, height, rgbd=rgbd, normals=False, panorama=panorama, num_props=P)
        on = _render("gallery", 2, width, height, rgbd=rgbd, normals=True, panorama=panorama, num_props=P)
        assert off["normal_row_bytes"] == 4 and on["normal_row_bytes"] == width * height * 4
        assert np.array_equal(on["depth"].view(np.uint32), off["depth"].view(np.uint32))
        assert np.array_equal(on["seg"], off["seg"])
        if rgbd:
            assert np.array_equal(on["rgb"], off["rgb"])
        assert np.array_equal((on["normals"] == 0).all(axis=-1), on["depth"] == 0)
        assert (on["normals"] != 0).any()


# ---- snapshots -----------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_normals_after_restore_equal_normals_at_save(monkeypatch):
    """render, save, step and render, restore, render: the restored scene gives the normals of
    the save"""
    from sims import make_executor
    W, props, width, height = 2, [30, 150], 48, 20
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", str(-(-sum(props) // W) + 64))
    ex = make_executor("gallery_sized", W, seed=3, rgbd=True, normals=True, props=props, width=width, height=height)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()

    def frame():
        ex.run(render)
        return ex.tensor(GALLERY_NORMALS, "int8", (2 * W, height, width, 4)).cpu().numpy().copy()
    for _ in range(3):
        ex.run(step)
    at_save = frame()
    assert (at_save != 0).any()
    with ex.snapshot() as snap:
        snap.save()
        for _ in range(5):
            ex.run(step)
        # the props turned: their normals moved
        assert not np.array_equal(frame(), at_save)
        snap.restore()
        assert np.array_equal(frame(), at_save)
    ex.close()


# ---- the C++ facade ------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_facade_normals_match_python_executor(tmp_path):
    exe = build_facade(tmp_path)
    assets, out = str(tmp_path / "assets.bin"), str(tmp_path / "frame.bin")
    _write_assets(assets)
    res = subprocess.run([exe, os.path.join(ROOT, "sims", "gallery", "sim.cpp"), assets, out],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    raw = np.fromfile(out, dtype=np.uint8)
    n = 2 * 2 * 64 * 32 * 4
    assert raw.size == 4 * n
    want = _render("gallery", 2, 64, 32, num_props=40)
    assert np.array_equal(raw[:n], want["rgb"].reshape(-1))
    assert np.array_equal(raw[n:2 * n], want["depth"].reshape(-1).view(np.uint8))
    assert np.array_equal(raw[2 * n:3 * n], want["seg"].reshape(-1).view(np.uint8))
    assert np.array_equal(raw[3 * n:], want["normals"].reshape(-1).view(np.uint8))
    assert (want["normals"] != 0).any(axis=-1).mean() > 0.3
