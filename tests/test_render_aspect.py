"""Non-square images in the batch ray caster: render_width x render_height pixels per view,
row-major [H][W], the vertical field of view over the H rows and the horizontal half-extent
widened by W / H (DESIGN 3.3).

GPU: every pixel against a brute-force float64 closest hit with the generalised camera rays,
colour restated from bvh_raycast.cpp (as tests/test_render_bvh.py does for squares), on both
instance paths (flat list at 40 props, TLAS at 100), RGBD and depth-only, wide, tall, thin and
one-row images; the textured colour model of tests/test_render_textures.py on a non-square
image; explicit square sizes against render_resolution, byte for byte; the C++ facade's
image-size overload against the Python-created executor.  Anywhere: config validation."""
import os
import struct
import subprocess

import numpy as np
import pytest

from sims.render_assets import GALLERY_MATERIALS, gallery_meshes
from test_render_bvh import _closest_hits, _quat_rotate, _world_triangles

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FOV_SCALE = 1.0 / np.tan(np.radians(70.0 * 0.5))
SIZES = [(64, 32), (32, 64), (40, 24), (37, 5), (256, 1), (24, 1)]


def camera_rays(pos, rot_inv, fov_scale, width, height):
    """bvh_raycast.cpp:58-88 in float64 with viewport_width = viewport_height * W / H and
    (px + 0.5) / W, (py + 0.5) / H: row-major [H * W, 3]"""
    q_inv = rot_inv.astype(np.float64)
    q = np.array([q_inv[0], -q_inv[1], -q_inv[2], -q_inv[3]])
    fwd = _quat_rotate(q, np.array([0.0, 1.0, 0.0]))
    fwd /= np.linalg.norm(fwd)
    u = _quat_rotate(q, np.array([1.0, 0.0, 0.0]))
    h = 1.0 / fov_scale
    vv = np.cross(fwd, u)
    vv /= np.linalg.norm(vv)
    horizontal, vertical = u * 2 * h * (width / height), vv * 2 * h
    ll = pos - horizontal / 2 - vertical / 2 + fwd
    pu = (np.arange(width) + 0.5) / width
    pv = (np.arange(height) + 0.5) / height
    d = ll[None, None] + pu[None, :, None] * horizontal + pv[:, None, None] * vertical - pos
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return d.reshape(-1, 3)


def test_camera_rays_reduce_to_the_square_model():
    from test_render_bvh import _camera_rays
    pos = np.array([0.3, -2.0, 1.5])
    q = np.array([0.9, 0.1, -0.3, 0.2])
    q /= np.linalg.norm(q)
    for res in (1, 7, 40):
        assert np.array_equal(camera_rays(pos, q, FOV_SCALE, res, res), _camera_rays(pos, q, FOV_SCALE, res))


def _render(name, W, P, width=None, height=None, resolution=None, rgbd=True, seed=5, **cfg):
    """3 steps + one render of a gallery fixture: exported columns, images, debug hit ids."""
    from sims import make_executor
    size = dict(width=width, height=height) if width is not None else dict(resolution=resolution)
    ex = make_executor(name, W, num_props=P, seed=seed, rgbd=rgbd, **size, **cfg)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(3):
        ex.run(step)
    ex.run(render)
    Wd = width if width is not None else resolution
    Hd = height if height is not None else resolution

    def col(slot, dtype, shape):
        return ex.tensor(slot, dtype, shape).cpu().numpy()
    out = dict(pos=col(0, "float32", (W, P, 3)), rot=col(1, "float32", (W, P, 4)),
               scale=col(2, "float32", (W, P, 3)), obj=col(3, "int32", (W, P)),
               mat=col(4, "int32", (W, P)), color=col(5, "uint32", (W, P)),
               vpos=col(6, "float32", (W, 2, 3)), vrot=col(7, "float32", (W, 2, 4)),
               depth=col(9, "float32", (2 * W, Hd, Wd)),
               hits=ex.renderDebugHits(2 * W, Hd, Wd).cpu().numpy(),
               row_bytes=(ex.exportedRowBytes(8), ex.exportedRowBytes(9)))
    if rgbd:
        out["rgb"] = col(8, "uint8", (2 * W, Hd, Wd, 4))
    ex.close()
    return out


def _check_against_brute_force(r, W, P, width, height):
    """ids, depth and colour of every pixel against the float64 oracle (tolerances of
    tests/test_render_bvh.py); returns (pixels, pixels hit, id-checked, colour-checked)"""
    import madrona_b200 as mb
    meshes = gallery_meshes()
    bvh = mb.MeshBVHData(meshes, gpu_id=-1)
    src_of = bvh.triangle_sources()
    first_tri = np.cumsum([0] + [len(m[1]) for m in meshes])
    total, hit_total, id_checked, rgb_checked = 0, 0, 0, 0
    for w in range(W):
        idx = np.array([i for i in range(P) if i == 0 or i % 17 != 0])     # the visible props
        obj_w, mat_w, col_w, rot_w = r["obj"][w, idx], r["mat"][w, idx], r["color"][w, idx], r["rot"][w, idx]
        tris, owner, src = _world_triangles(meshes, r["pos"][w, idx], rot_w, r["scale"][w, idx], obj_w)
        for v in range(2):
            view = 2 * w + v
            cam = r["vpos"][w, v].astype(np.float64) + np.array([0.0, 0.0, 0.25])
            q = r["vrot"][w, v].astype(np.float64)
            rays = camera_rays(cam, np.array([q[0], -q[1], -q[2], -q[3]]), FOV_SCALE, width, height)
            o = np.broadcast_to(cam, rays.shape)
            t, tri, t2 = _closest_hits(o, rays, tris)
            want_hit = np.isfinite(t)
            got_d = r["depth"][view].reshape(-1)
            got_hit = got_d > 0
            total += len(t)
            # silhouettes may differ between the watertight fp32 test and float64 Moeller-Trumbore
            assert (want_hit != got_hit).sum() <= max(1, int(0.005 * len(t))), (w, v)
            both = want_hit & got_hit
            hit_total += int(both.sum())
            np.testing.assert_allclose(got_d[both], t[both], rtol=1e-4, atol=1e-4)
            with np.errstate(invalid="ignore"):
                clear = both & ((t2 - t) > 1e-3 * np.maximum(t, 1.0))
            g_inst, g_tri = r["hits"][view].reshape(-1, 2)[:, 0], r["hits"][view].reshape(-1, 2)[:, 1]
            assert ((g_inst >= 0) == got_hit).all()
            want_inst = owner[np.maximum(tri, 0)]
            assert np.array_equal(g_inst[clear], want_inst[clear])
            got_src = src_of[first_tri[obj_w[want_inst]] + np.maximum(g_tri, 0)]
            assert np.array_equal(got_src[clear], src[np.maximum(tri, 0)][clear])
            id_checked += int(clear.sum())
            if "rgb" not in r:
                continue

            # colour: bvh_raycast.cpp:756-938 on the brute-force hit (see tests/test_render_bvh.py)
            sel = np.nonzero(clear)[0]
            inst_k = want_inst[sel]
            n_obj = []
            for k, s_tri in zip(inst_k, src[tri[sel]]):
                vtx, f, _ = meshes[int(obj_w[k])]
                a, b, c = vtx[f[s_tri]].astype(np.float64)
                nn = np.cross(b - a, c - a)
                n_obj.append(_quat_rotate(rot_w[k].astype(np.float64), nn / np.linalg.norm(nn)))
            n = np.array(n_obj).reshape(-1, 3)
            hit_pos = o[sel] + t[sel, None] * rays[sel]
            ldir = -np.array([0.3, 0.2, -0.9327379])
            facing = (n @ ldir) > 0
            st = _closest_hits(hit_pos + 1e-3 * n, np.broadcast_to(ldir, hit_pos.shape), tris, t_min=1e-6)[0]
            st_a = _closest_hits(hit_pos + 3e-3 * n, np.broadcast_to(ldir, hit_pos.shape), tris, t_min=1e-6)[0]
            st_b = _closest_hits(hit_pos + 3e-4 * n, np.broadcast_to(ldir, hit_pos.shape), tris, t_min=1e-6)[0]
            graze = (np.isfinite(st) != np.isfinite(st_a)) | (np.isfinite(st) != np.isfinite(st_b))
            contrib = np.where(facing & ~np.isfinite(st), np.clip(n @ ldir, 0, 1), 0.0)
            to_l = np.array([0.0, 0.0, 9.0]) - hit_pos
            to_l /= np.linalg.norm(to_l, axis=1, keepdims=True)
            ang = np.arccos(np.clip((-to_l) @ np.array([0.0, 0.0, -1.0]), -1, 1))
            contrib += np.where(np.abs(ang) <= 0.9, np.clip((n * to_l).sum(1), 0, 1), 0.0)
            base = np.ones((len(sel), 3))
            for j, k in enumerate(inst_k):
                m = int(mat_w[k])
                if m == -2:
                    hx = int(col_w[k])
                    base[j] = [((hx >> 16) & 255) / 255.0, ((hx >> 8) & 255) / 255.0, (hx & 255) / 255.0]
                else:
                    if m == -1:
                        m = meshes[int(obj_w[k])][2]
                    if m >= 0:
                        base[j] = GALLERY_MATERIALS[m, :3]
            want_rgb = np.clip(np.maximum(0.2, contrib)[:, None] * base, 0, 1) * 255.0
            got_rgb = r["rgb"][view].reshape(-1, 4)[sel, :3].astype(np.float64)
            edge = graze | (np.abs(np.abs(ang) - 0.9) < 5e-3) | (np.abs(n @ ldir) < 5e-3)
            # within +-1 of the float64 colour (the 8-bit conversion truncates)
            ok = np.abs(got_rgb - want_rgb).max(axis=1) <= 1.0 + 1e-9
            assert ok[~edge].mean() > 0.99, (w, v, float(ok[~edge].mean()), int((~edge).sum()))
            assert (r["rgb"][view][..., 3] == 255).all()
            rgb_checked += int((~edge).sum())
    return total, hit_total, id_checked, rgb_checked


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_instances", "flat_list_40_instances"])
def test_gpu_non_square_pixels_match_brute_force(monkeypatch, P, size):
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    width, height = size
    # one-row images look along the horizon, where most rays miss: more worlds for more hits
    W = 4 if height < 4 else 1
    r = _render("gallery", W, P, width=width, height=height)
    assert r["row_bytes"] == (width * height * 4, width * height * 4)
    total, hit_total, id_checked, rgb_checked = _check_against_brute_force(r, W, P, width, height)
    assert hit_total > (0.3 * total if height >= 4 else 16)
    assert id_checked > 0.7 * hit_total
    assert rgb_checked > 0.5 * id_checked
    # depth-only: the same depth and hits, bit for bit
    d = _render("gallery", W, P, width=width, height=height, rgbd=False)
    assert d["row_bytes"] == r["row_bytes"]
    assert np.array_equal(d["depth"].view(np.uint32), r["depth"].view(np.uint32))
    assert np.array_equal(d["hits"], r["hits"])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_instances", "flat_list_40_instances"])
def test_gpu_explicit_square_size_matches_render_resolution_byte_for_byte(monkeypatch, P):
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    for rgbd in (True, False):
        a = _render("gallery", 2, P, resolution=40, rgbd=rgbd)
        b = _render("gallery", 2, P, width=40, height=40, rgbd=rgbd)
        assert a["row_bytes"] == b["row_bytes"] == (40 * 40 * 4, 40 * 40 * 4)
        assert np.array_equal(a["depth"].view(np.uint32), b["depth"].view(np.uint32))
        assert np.array_equal(a["hits"], b["hits"])
        assert (a["depth"] > 0).mean() > 0.3
        if rgbd:
            assert np.array_equal(a["rgb"], b["rgb"])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_instances", "flat_list_40_instances"])
def test_gpu_textured_non_square_colour_matches_filter_model(monkeypatch, P):
    import test_render_textures as trt
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    width, height, W = 48, 20, 3
    # the textured oracle of tests/test_render_textures.py, its camera rays made non-square
    monkeypatch.setattr(trt, "_camera_rays", lambda pos, rot_inv, fov, res: camera_rays(pos, rot_inv, fov, width,
                                                                                         height))
    cover = {k: 0 for k in ("texture_0", "texture_1", "texture_2", "override_textured", "override_colour",
                            "ground_wrapped")}
    r = _render("gallery_textured", W, P, width=width, height=height)
    checked = trt._check_textured_colour(r, W, P, None, False, cover)
    assert checked > 1000
    assert cover["texture_0"] > 0 and cover["texture_1"] > 0, cover


# ---- config validation (checked before any CUDA call, so it runs without a GPU too) -------------

INVALID = [
    (0, 64, 0, "render_width and render_height must be set together"),
    (0, 0, 32, "render_width and render_height must be set together"),
    (40, 64, 32, "contradicts render_resolution = 40"),
    (40, 40, 41, "contradicts render_resolution = 40"),
    (0, 65536, 16384, "exceed the 32-bit component size"),
    (32768, 0, 0, "exceed the 32-bit component size"),
]


def _create_with(monkeypatch, resolution, width, height):
    from madrona_b200.executor import _MaterialViewC, _MeshBVHViewC, _RenderConfigC
    from sims import SIMS, make_executor
    rc = _RenderConfigC(0, _MeshBVHViewC(), _MaterialViewC(), resolution, 0.001, 1000.0, width, height)
    monkeypatch.setattr(SIMS["gallery"], "render", lambda cfg: (rc, None))
    return make_executor("gallery", 2, num_props=8)


@pytest.mark.parametrize("resolution,width,height,message", INVALID)
def test_invalid_image_size_is_rejected_at_creation(monkeypatch, resolution, width, height, message):
    import madrona_b200 as mb
    with pytest.raises(mb.MadronaB200Error, match=message):
        _create_with(monkeypatch, resolution, width, height)


@pytest.mark.gpu
def test_gpu_device_is_healthy_after_rejected_configs(monkeypatch):
    import torch
    import madrona_b200 as mb
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    with monkeypatch.context() as m:
        for resolution, width, height, message in INVALID:
            with pytest.raises(mb.MadronaB200Error, match=message):
                _create_with(m, resolution, width, height)
    r = _render("gallery", 2, 40, width=37, height=5)
    torch.cuda.synchronize()
    assert (r["depth"] > 0).mean() > 0.3
    assert r["row_bytes"] == (37 * 5 * 4, 37 * 5 * 4)


# ---- the C++ facade's image-size overload ------------------------------------------------------

def _write_assets(path):
    meshes = gallery_meshes()
    with open(path, "wb") as f:
        f.write(struct.pack("<I", len(meshes)))
        for pos, tris, mat in meshes:
            f.write(struct.pack("<IIi", len(pos), len(tris), mat))
            f.write(np.ascontiguousarray(pos, dtype="<f4").tobytes())
            f.write(np.ascontiguousarray(tris, dtype="<u4").tobytes())
        f.write(struct.pack("<I", len(GALLERY_MATERIALS)))
        f.write(np.ascontiguousarray(GALLERY_MATERIALS, dtype="<f4").tobytes())     # == mb2_source_material


def _build_facade(tmp_path):
    exe = str(tmp_path / "facade_render_aspect")
    cmd = ["g++", "-std=c++20", "-O1", "-I" + os.path.join(ROOT, "madrona_b200", "host"),
           os.path.join(ROOT, "tests", "cpp", "facade_render_aspect.cpp"), "-o", exe,
           "-L" + os.path.join(ROOT, "madrona_b200"), "-lmadrona_b200",
           "-Wl,-rpath," + os.path.join(ROOT, "madrona_b200"),
           "-L/usr/local/cuda/lib64", "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    return exe


def test_facade_image_size_overload_compiles(tmp_path):
    _build_facade(tmp_path)


@pytest.mark.gpu
def test_gpu_facade_image_size_overload_matches_python_executor(monkeypatch, tmp_path):
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    exe = _build_facade(tmp_path)
    assets, out = str(tmp_path / "assets.bin"), str(tmp_path / "frame.bin")
    _write_assets(assets)
    res = subprocess.run([exe, os.path.join(ROOT, "sims", "gallery", "sim.cpp"), assets, out],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    raw = np.fromfile(out, dtype=np.uint8)
    n = 2 * 2 * 64 * 32 * 4
    assert raw.size == 2 * n
    want = _render("gallery", 2, 40, width=64, height=32)
    assert np.array_equal(raw[:n], want["rgb"].reshape(-1))
    assert np.array_equal(raw[n:], want["depth"].reshape(-1).view(np.uint8))
    assert (want["depth"] > 0).mean() > 0.3
