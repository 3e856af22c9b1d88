"""Panoramic views in the batch ray caster (mb2_render_config::projection = 1, DESIGN 3.3): every
view's W x H image covers 360 degrees of azimuth across its columns and the vertical field of
view across its rows, evenly spaced in elevation; depth is the distance along the unit ray.

GPU: every pixel's debug (instance, triangle), depth and segmentation against the float64
brute-force closest hit along the panorama ray, on the flat list (40 props), the TLAS (100
props) and the large-world TLAS builder (a world of 150 props), at 256 x 16, 37 x 5 and 360 x 1;
the panorama sees props behind the camera that the pinhole misses; colour, untextured (lights
and shadow rays on) and textured, against the oracles of tests/test_render_aspect.py and
tests/test_render_textures.py with their camera rays swapped for panorama rays; ids after
room_render resets; the C++ facade's RenderProjection overload against the Python-created
executor.  The float32 ray formula and the culls are modelled in
tests/test_raycast_panorama_model.py."""
import os
import subprocess

import numpy as np
import pytest

from sims.render_assets import gallery_meshes
from test_raycast_panorama_model import build_facade
from test_render_aspect import FOV_SCALE, _write_assets, camera_rays
from test_render_bvh import _closest_hits, _quat_rotate, _world_triangles

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GALLERY_RGB, GALLERY_DEPTH, GALLERY_PROP_ENTITY, GALLERY_SEG = 8, 9, 10, 11
ROOM_BODY_ENTITY, ROOM_DEPTH, ROOM_AGENT_ENTITY, ROOM_SEG = 11, 14, 17, 18


def panorama_rays(pos, rot_inv, fov_scale, width, height):
    """the panorama's primary rays in float64, row-major [H * W, 3]: the view frame of
    tests/test_render_aspect.py's camera_rays, azimuth over the columns and elevation over the
    rows (DESIGN 3.3)"""
    q_inv = rot_inv.astype(np.float64)
    q = np.array([q_inv[0], -q_inv[1], -q_inv[2], -q_inv[3]])
    fwd = _quat_rotate(q, np.array([0.0, 1.0, 0.0]))
    fwd /= np.linalg.norm(fwd)
    u = _quat_rotate(q, np.array([1.0, 0.0, 0.0]))
    vv = np.cross(fwd, u)
    vv /= np.linalg.norm(vv)
    h = 1.0 / fov_scale
    phi_max = np.arctan(h)
    s = -1.0 if h < 0 else 1.0
    theta = s * 2 * np.pi * ((np.arange(width) + 0.5) / width - 0.5)
    phi = 2 * phi_max * ((np.arange(height) + 0.5) / height - 0.5)
    cp, sp = np.cos(phi)[:, None, None], np.sin(phi)[:, None, None]
    d = cp * (np.cos(theta)[None, :, None] * fwd + np.sin(theta)[None, :, None] * u) + sp * vv
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return d.reshape(-1, 3)


def test_panorama_rays_centre_on_the_pinhole_axis():
    pos = np.array([0.3, -2.0, 1.5])
    q = np.array([0.9, 0.1, -0.3, 0.2])
    q /= np.linalg.norm(q)
    pano = panorama_rays(pos, q, FOV_SCALE, 9, 5).reshape(5, 9, 3)
    pin = camera_rays(pos, q, FOV_SCALE, 9, 5).reshape(5, 9, 3)
    np.testing.assert_allclose(pano[2, 4], pin[2, 4], atol=1e-12)
    # one row: the horizon, every direction
    ring = panorama_rays(pos, q, FOV_SCALE, 360, 1)
    vv = np.cross(pin[2, 4], _quat_rotate(np.array([q[0], -q[1], -q[2], -q[3]]), np.array([1.0, 0.0, 0.0])))
    assert np.abs(ring @ vv).max() < 1e-12


def _visible(P):
    """prop rows of a gallery world that are drawn: the ground and all but every 17th prop"""
    return np.array([i for i in range(P) if i == 0 or i % 17 != 0], dtype=np.int64)


def _render(name, W, width, height, steps=3, rgbd=True, **cfg):
    """`steps` steps of a gallery fixture, then one panoramic frame with segmentation; flat
    exported columns (rows of all worlds)"""
    from sims import make_executor
    ex = make_executor(name, W, rgbd=rgbd, segmentation=True, panorama=True, seed=5, width=width, height=height,
                       **cfg)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(steps):
        ex.run(step)
    ex.run(render)
    rows = ex.exportedNumRows(0)

    def col(slot, dtype, shape):
        return ex.tensor(slot, dtype, shape).cpu().numpy().copy()
    out = dict(rows=rows, depth=col(GALLERY_DEPTH, "float32", (2 * W, height, width)),
               seg=col(GALLERY_SEG, "int32", (2 * W, height, width)),
               entity=col(GALLERY_PROP_ENTITY, "int32", (rows, 2))[:, 1],
               pos=col(0, "float32", (rows, 3)), rot=col(1, "float32", (rows, 4)),
               scale=col(2, "float32", (rows, 3)), obj=col(3, "int32", (rows,)),
               vpos=col(6, "float32", (W, 2, 3)), vrot=col(7, "float32", (W, 2, 4)))
    if rgbd:
        out["rgb"] = col(GALLERY_RGB, "uint8", (2 * W, height, width, 4))
    if os.environ.get("MADRONA_B200_RENDER_DEBUG") == "1":
        out["hits"] = ex.renderDebugHits(2 * W, height, width).cpu().numpy()
    ex.close()
    return out


# ---- every pixel against the float64 brute-force closest hit -----------------------------------------

CASES = {
    "flat_list_40_props": ("gallery", dict(num_props=40), [40] * 3),
    "tlas_100_props": ("gallery", dict(num_props=100), [100] * 3),
    # world 0: 142 visible props, past the warp builder's 128 (the large-world TLAS builder);
    # world 1 on the flat list
    "large_tlas_150_props": ("gallery_sized", dict(props=[150, 40]), [150, 40]),
}
SIZES = [(256, 16), (37, 5), (360, 1)]      # (width, height)


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
@pytest.mark.parametrize("case", sorted(CASES))
def test_gpu_panorama_pixels_match_brute_force(monkeypatch, case, size):
    import madrona_b200 as mb
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    name, cfg, props = CASES[case]
    W = len(props)
    width, height = size
    if name == "gallery_sized":
        # tables with room for every prop from the start (tests/test_render_large_worlds.py)
        monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", str(-(-sum(props) // W) + 64))
    r = _render(name, W, width, height, **cfg)
    assert r["rows"] == sum(props)
    meshes = gallery_meshes()
    src_of = mb.MeshBVHData(meshes, gpu_id=-1).triangle_sources()
    first_tri = np.cumsum([0] + [len(m[1]) for m in meshes])
    starts = np.concatenate([[0], np.cumsum(props)[:-1]])
    total = hit_total = id_checked = 0
    behind_only = 0          # props the panorama shows behind the camera that the pinhole misses
    for w in range(W):
        rows = starts[w] + _visible(props[w])
        obj_w, ids_w = r["obj"][rows], r["entity"][rows]
        tris, owner, src = _world_triangles(meshes, r["pos"][rows], r["rot"][rows], r["scale"][rows], obj_w)
        for v in range(2):
            view = 2 * w + v
            cam = r["vpos"][w, v].astype(np.float64) + np.array([0.0, 0.0, 0.25])
            q = r["vrot"][w, v].astype(np.float64)
            q_inv = np.array([q[0], -q[1], -q[2], -q[3]])
            rays = panorama_rays(cam, q_inv, FOV_SCALE, width, height)
            t, tri, t2 = _closest_hits(np.broadcast_to(cam, rays.shape), rays, tris)
            want_hit = np.isfinite(t)
            got_d = r["depth"][view].reshape(-1)
            got_hit = got_d > 0
            seg = r["seg"][view].reshape(-1)
            g_inst, g_tri = r["hits"][view].reshape(-1, 2)[:, 0], r["hits"][view].reshape(-1, 2)[:, 1]
            total += len(t)
            # silhouettes may differ between the watertight fp32 test and float64 Moeller-Trumbore
            assert (want_hit != got_hit).sum() <= max(1, int(0.005 * len(t))), (case, w, v)
            both = want_hit & got_hit
            hit_total += int(both.sum())
            np.testing.assert_allclose(got_d[both], t[both], rtol=1e-4, atol=1e-4)
            assert ((g_inst >= 0) == got_hit).all()
            with np.errstate(invalid="ignore"):
                clear = both & ((t2 - t) > 1e-3 * np.maximum(t, 1.0))
            want_inst = owner[np.maximum(tri, 0)]
            assert np.array_equal(g_inst[clear], want_inst[clear]), (case, w, v)
            got_src = src_of[first_tri[obj_w[want_inst]] + np.maximum(g_tri, 0)]
            assert np.array_equal(got_src[clear], src[np.maximum(tri, 0)][clear]), (case, w, v)
            id_checked += int(clear.sum())
            # segmentation: the debug instance's entity, -1 exactly where the depth is 0
            assert np.array_equal(seg[got_hit], ids_w[g_inst[got_hit]]), (case, w, v)
            assert np.array_equal(seg == -1, got_d == 0)
            # what the pinhole of the same view sees
            pin = camera_rays(cam, q_inv, FOV_SCALE, 40, 40)
            pt = _closest_hits(np.broadcast_to(cam, pin.shape), pin, tris)[1]
            pin_seen = set(owner[pt[pt >= 0]].tolist())
            behind_only += len(set(g_inst[got_hit].tolist()) - pin_seen)
    if height >= 4:
        assert hit_total > 0.25 * total
    else:
        assert hit_total > 16
    assert id_checked > 0.7 * hit_total
    assert behind_only > 0


# ---- colour ------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_instances", "flat_list_40_instances"])
def test_gpu_panorama_colour_matches_brute_force(monkeypatch, P):
    """tests/test_render_aspect.py's oracle (ids, depth, colour with both lights and shadow
    rays) with its camera rays swapped for panorama rays"""
    import test_render_aspect as tra
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    width, height, W = 128, 16, 2
    monkeypatch.setattr(tra, "camera_rays", panorama_rays)
    r = tra._render("gallery", W, P, width=width, height=height, panorama=True)
    total, hit_total, id_checked, rgb_checked = tra._check_against_brute_force(r, W, P, width, height)
    assert hit_total > 0.25 * total
    assert id_checked > 0.7 * hit_total
    assert rgb_checked > 0.5 * id_checked


@pytest.mark.gpu
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_instances", "flat_list_40_instances"])
def test_gpu_panorama_textured_colour_matches_filter_model(monkeypatch, P):
    import test_render_aspect as tra
    import test_render_textures as trt
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    width, height, W = 96, 20, 3
    # the textured oracle of tests/test_render_textures.py, its camera rays made panoramic
    monkeypatch.setattr(trt, "_camera_rays", lambda pos, rot_inv, fov, res: panorama_rays(pos, rot_inv, fov, width,
                                                                                           height))
    cover = {k: 0 for k in ("texture_0", "texture_1", "texture_2", "override_textured", "override_colour",
                            "ground_wrapped")}
    r = tra._render("gallery_textured", W, P, width=width, height=height, panorama=True)
    checked = trt._check_textured_colour(r, W, P, None, False, cover)
    assert checked > 1000
    assert cover["texture_0"] > 0 and cover["texture_1"] > 0, cover


# ---- ids after resets ----------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_room_panorama_ids_are_live_renderables_of_the_view_world_across_resets():
    """room_render with panoramic views (a 64 x 8 ring around each agent) across resets that
    destroy and recreate its cubes: every id a world's views show is one of that world's live
    renderable entities (its 2 agents and 31 bodies)"""
    from sims import make_executor
    from trace_utils import make_inputs
    import torch
    W, steps, width, height, bodies = 4, 14, 64, 8, 31
    ins = make_inputs("room", W, steps, seed=4)
    ex = make_executor("room_render", W, episode_len=5, seed=3, width=width, height=height, rgbd=True,
                       segmentation=True, panorama=True)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    in_t = {"reset": ex.tensor(0, "int32", (W, 1)), "action": ex.tensor(1, "int32", (W, 2, 3))}
    first = None
    changed = False
    for t in range(steps):
        for name, arr in ins.items():
            in_t[name].copy_(torch.from_numpy(np.ascontiguousarray(arr[t])))
        torch.cuda.synchronize()
        ex.run(step)
        ex.run(render)
        body = ex.tensor(ROOM_BODY_ENTITY, "int32", (W * bodies, 2)).cpu().numpy().reshape(W, bodies, 2)
        agent = ex.tensor(ROOM_AGENT_ENTITY, "int32", (W, 2, 2)).cpu().numpy()
        seg = ex.tensor(ROOM_SEG, "int32", (2 * W, height, width)).cpu().numpy()
        depth = ex.tensor(ROOM_DEPTH, "float32", (2 * W, height, width)).cpu().numpy()
        handles = {tuple(e) for e in body.reshape(-1, 2).tolist()}
        if first is None:
            first = handles
        changed = changed or handles != first
        assert np.array_equal(seg == -1, depth == 0)
        for w in range(W):
            live = set(body[w, :, 1].tolist()) | set(agent[w, :, 1].tolist())
            shown = set(np.unique(seg[2 * w:2 * w + 2]).tolist()) - {-1}
            assert shown and shown <= live, (t, w, sorted(shown - live))
    assert changed, "no reset recreated an entity"
    ex.close()


# ---- the C++ facade's overload ---------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_facade_panorama_overload_matches_python_executor(tmp_path):
    exe = build_facade(tmp_path)
    assets, out = str(tmp_path / "assets.bin"), str(tmp_path / "frame.bin")
    _write_assets(assets)
    res = subprocess.run([exe, os.path.join(ROOT, "sims", "gallery", "sim.cpp"), assets, out],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    raw = np.fromfile(out, dtype=np.uint8)
    n = 2 * 2 * 256 * 16 * 4
    assert raw.size == 3 * n
    want = _render("gallery", 2, 256, 16, num_props=40)
    assert np.array_equal(raw[:n], want["rgb"].reshape(-1))
    assert np.array_equal(raw[n:2 * n], want["depth"].reshape(-1).view(np.uint8))
    assert np.array_equal(raw[2 * n:], want["seg"].reshape(-1).view(np.uint8))
    assert (want["seg"] >= 0).mean() > 0.25
