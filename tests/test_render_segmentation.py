"""Segmentation output of the batch ray caster (mb2_render_config::segmentation, DESIGN 3.3):
every view gets a row-major [H][W] int32 image holding the Entity id of the renderable that the
pixel's primary ray hits first, -1 where it hits nothing.

GPU: every pixel against the debug hit buffer's instance (instance k of world w = the k-th
visible prop row of w, as in tests/test_render_bvh.py) on the flat list (40 props), the TLAS
(100 props) and the large-world TLAS builder (a world above 128 props); against the float64
brute-force closest hit; RGB and depth byte-identical with the output on and off; ids after
resets reuse entities; snapshots; the C++ facade's overload against the Python-created
executor.  Anywhere: the C ABI layout and config validation."""
import os
import subprocess

import numpy as np
import pytest

from sims.render_assets import gallery_meshes
from test_render_aspect import FOV_SCALE, _write_assets, camera_rays
from test_render_bvh import _closest_hits, _world_triangles

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GALLERY_RGB, GALLERY_DEPTH, GALLERY_PROP_ENTITY, GALLERY_SEG = 8, 9, 10, 11
ROOM_BODY_ENTITY, ROOM_RGB, ROOM_DEPTH, ROOM_AGENT_ENTITY, ROOM_SEG = 11, 13, 14, 17, 18


def _visible(P):
    """prop rows of a gallery world that are drawn: the ground and all but every 17th prop"""
    return np.array([i for i in range(P) if i == 0 or i % 17 != 0], dtype=np.int64)


def _render(name, W, steps=4, width=None, height=None, resolution=40, rgbd=True, segmentation=True, **cfg):
    """`steps` steps of a gallery fixture (the props spin and bob), then one frame"""
    from sims import make_executor
    size = dict(width=width, height=height) if width is not None else dict(resolution=resolution)
    Wd = width if width is not None else resolution
    Hd = height if height is not None else resolution
    ex = make_executor(name, W, rgbd=rgbd, segmentation=segmentation, seed=5, **size, **cfg)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(steps):
        ex.run(step)
    ex.run(render)
    rows = ex.exportedNumRows(0)

    def col(slot, dtype, shape):
        return ex.tensor(slot, dtype, shape).cpu().numpy().copy()
    out = dict(rows=rows, depth=col(GALLERY_DEPTH, "float32", (2 * W, Hd, Wd)),
               entity=col(GALLERY_PROP_ENTITY, "int32", (rows, 2))[:, 1],
               seg_row_bytes=ex.exportedRowBytes(GALLERY_SEG))
    if rgbd:
        out["rgb"] = col(GALLERY_RGB, "uint8", (2 * W, Hd, Wd, 4))
    if segmentation:
        out["seg"] = col(GALLERY_SEG, "int32", (2 * W, Hd, Wd))
    if os.environ.get("MADRONA_B200_RENDER_DEBUG") == "1":
        out["hits"] = ex.renderDebugHits(2 * W, Hd, Wd).cpu().numpy()
        out.update(pos=col(0, "float32", (rows, 3)), rot=col(1, "float32", (rows, 4)),
                   scale=col(2, "float32", (rows, 3)), obj=col(3, "int32", (rows,)),
                   vpos=col(6, "float32", (W, 2, 3)), vrot=col(7, "float32", (W, 2, 4)))
    ex.close()
    return out


# ---- exact, every pixel, against the debug hit buffer ------------------------------------------

EXACT = {
    "flat_list_40_props": ("gallery", 3, dict(num_props=40), [40] * 3),
    "tlas_100_props": ("gallery", 3, dict(num_props=100), [100] * 3),
    # world 0: 142 visible props, past the warp builder's 128 (the large-world TLAS builder);
    # world 1 on the flat list
    "large_tlas_150_props": ("gallery_sized", 2, dict(props=[150, 40]), [150, 40]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(EXACT))
def test_gpu_segmentation_is_the_hit_instance_entity_on_every_pixel(monkeypatch, case):
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    name, W, cfg, props = EXACT[case]
    if name == "gallery_sized":
        # tables with room for every prop from the start (tests/test_render_large_worlds.py)
        monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", str(-(-sum(props) // W) + 64))
    r = _render(name, W, steps=5, **cfg)
    assert r["rows"] == sum(props)
    assert r["seg_row_bytes"] == 40 * 40 * 4
    starts = np.concatenate([[0], np.cumsum(props)[:-1]])
    all_ids = set(r["entity"].tolist())
    assert len(all_ids) == sum(props)           # ids are unique among live entities
    hit_pixels = 0
    for w in range(W):
        rows_w = starts[w] + np.arange(props[w])
        vis = _visible(props[w])
        ids_w = r["entity"][rows_w[vis]]                        # instance k -> entity id
        hidden = set(r["entity"][np.setdiff1d(rows_w, rows_w[vis])].tolist())
        others = all_ids - set(r["entity"][rows_w].tolist())
        for v in (2 * w, 2 * w + 1):
            seg = r["seg"][v].reshape(-1)
            inst = r["hits"][v].reshape(-1, 2)[:, 0]
            hit = inst >= 0
            assert (inst < len(ids_w)).all()
            assert np.array_equal(seg[hit], ids_w[inst[hit]]), (case, w, v)
            assert (seg[~hit] == -1).all()
            assert np.array_equal(seg == -1, r["depth"][v].reshape(-1) == 0)
            got = set(np.unique(seg[hit]).tolist())
            assert not got & hidden, (case, w, v)
            assert not got & others, (case, w, v)
            hit_pixels += int(hit.sum())
    assert hit_pixels > 0.3 * 2 * W * 40 * 40


# ---- against the float64 brute-force closest hit --------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_props", "flat_list_40_props"])
def test_gpu_segmentation_matches_brute_force_closest_hit(monkeypatch, P):
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    W, width, height = 2, 48, 20
    r = _render("gallery", W, steps=3, width=width, height=height, num_props=P)
    meshes = gallery_meshes()
    checked = total = 0
    for w in range(W):
        rows = w * P + _visible(P)
        ids_w = r["entity"][rows]
        tris, owner, _src = _world_triangles(meshes, r["pos"][rows], r["rot"][rows], r["scale"][rows],
                                             r["obj"][rows])
        for v in range(2):
            view = 2 * w + v
            cam = r["vpos"][w, v].astype(np.float64) + np.array([0.0, 0.0, 0.25])
            q = r["vrot"][w, v].astype(np.float64)
            rays = camera_rays(cam, np.array([q[0], -q[1], -q[2], -q[3]]), FOV_SCALE, width, height)
            t, tri, t2 = _closest_hits(np.broadcast_to(cam, rays.shape), rays, tris)
            seg = r["seg"][view].reshape(-1)
            want_hit = np.isfinite(t)
            total += len(t)
            # silhouettes may differ between the watertight fp32 test and float64 Moeller-Trumbore
            assert (want_hit != (seg >= 0)).sum() <= max(1, int(0.005 * len(t)))
            with np.errstate(invalid="ignore"):
                clear = want_hit & (seg >= 0) & ((t2 - t) > 1e-3 * np.maximum(t, 1.0))
            want = ids_w[owner[np.maximum(tri, 0)]]
            assert np.array_equal(seg[clear], want[clear]), (P, w, v)
            checked += int(clear.sum())
    assert checked > 0.25 * total


# ---- the other outputs do not change ---------------------------------------------------------------

SIZES = [(40, 40), (64, 32), (37, 5), (256, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_props", "flat_list_40_props"])
def test_gpu_rgb_and_depth_are_byte_identical_with_segmentation_on_and_off(P, size):
    width, height = size
    kw = dict(resolution=40) if width == height else dict(width=width, height=height)
    W = 4 if height < 4 else 2
    for rgbd in (True, False):
        off = _render("gallery", W, steps=3, rgbd=rgbd, segmentation=False, num_props=P, **kw)
        on = _render("gallery", W, steps=3, rgbd=rgbd, segmentation=True, num_props=P, **kw)
        assert off["seg_row_bytes"] == 4 and on["seg_row_bytes"] == width * height * 4
        assert np.array_equal(on["depth"].view(np.uint32), off["depth"].view(np.uint32))
        if rgbd:
            assert np.array_equal(on["rgb"], off["rgb"])
        assert np.array_equal(on["seg"] == -1, on["depth"] == 0)
        assert (on["seg"] >= 0).any()


# ---- ids after resets --------------------------------------------------------------------------------

@pytest.mark.gpu
def test_gpu_room_ids_are_live_renderables_of_the_view_world_across_resets():
    """room_render destroys and recreates its cubes at every reset (short episodes here), so
    entity ids are freed and handed out again; after every step each id a world's views show
    is one of that world's live renderable entities (its 2 agents and 31 bodies)."""
    from sims import make_executor
    from trace_utils import make_inputs
    import torch
    W, steps, res, bodies = 4, 14, 32, 31
    ins = make_inputs("room", W, steps, seed=4)
    ex = make_executor("room_render", W, episode_len=5, seed=3, resolution=res, rgbd=True, segmentation=True)
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
        assert ex.exportedNumRows(ROOM_BODY_ENTITY) == W * bodies
        body = ex.tensor(ROOM_BODY_ENTITY, "int32", (W * bodies, 2)).cpu().numpy().reshape(W, bodies, 2)
        agent = ex.tensor(ROOM_AGENT_ENTITY, "int32", (W, 2, 2)).cpu().numpy()
        seg = ex.tensor(ROOM_SEG, "int32", (2 * W, res, res)).cpu().numpy()
        depth = ex.tensor(ROOM_DEPTH, "float32", (2 * W, res, res)).cpu().numpy()
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


# ---- snapshots -----------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("sim,cfg", [
    ("gallery_sized", {"props": [30, 150], "width": 48, "height": 20}),
    ("room_render", {"episode_len": 12, "resolution": 32}),
])
def test_gpu_segmentation_after_restore_equals_segmentation_at_save(monkeypatch, sim, cfg):
    """render, save, step and render, restore, render: the restored instance list (80-byte
    records with their entity ids) gives the segmentation of the save"""
    import torch
    from sims import make_executor
    from trace_utils import make_inputs
    gallery = sim.startswith("gallery")
    W = 2 if gallery else 4
    (seg_slot, depth_slot), h, w = ((GALLERY_SEG, GALLERY_DEPTH), 20, 48) if gallery else ((ROOM_SEG, ROOM_DEPTH), 32, 32)
    if gallery:
        monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", str(-(-sum(cfg["props"]) // W) + 64))
    ex = make_executor(sim, W, seed=3, rgbd=True, segmentation=True, **cfg)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    ins = {} if gallery else make_inputs("room", W, 8, seed=1)
    in_t = {} if gallery else {"reset": ex.tensor(0, "int32", (W, 1)), "action": ex.tensor(1, "int32", (W, 2, 3))}

    def advance(t):
        for name, arr in ins.items():
            in_t[name].copy_(torch.from_numpy(np.ascontiguousarray(arr[t])))
        torch.cuda.synchronize()
        ex.run(step)

    def frame():
        """(segmentation, depth) of a new frame"""
        ex.run(render)
        return (ex.tensor(seg_slot, "int32", (2 * W, h, w)).cpu().numpy().copy(),
                ex.tensor(depth_slot, "float32", (2 * W, h, w)).cpu().numpy().copy())
    for t in range(3):
        advance(t)
    seg_at_save, depth_at_save = frame()
    assert (seg_at_save >= 0).any()
    with ex.snapshot() as snap:
        snap.save()
        for t in range(3, 8):
            advance(t)
        # the scene moved (the ids a view shows may not have changed)
        assert not np.array_equal(frame()[1], depth_at_save)
        snap.restore()
        seg, depth = frame()
        assert np.array_equal(seg, seg_at_save)
        assert np.array_equal(depth, depth_at_save)
    ex.close()


# ---- config validation and the C ABI (no GPU needed) -------------------------------------------------

def test_render_config_matches_the_c_header(tmp_path):
    import ctypes
    from madrona_b200.executor import _RenderConfigC
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "madrona_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", sizeof(mb2_render_config), '
                   'offsetof(mb2_render_config, segmentation), offsetof(mb2_render_config, render_height));'
                   ' return 0; }\n')
    exe = str(tmp_path / "layout")
    res = subprocess.run(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    size, seg_at, height_at = (int(x) for x in subprocess.run([exe], capture_output=True, text=True,
                                                              check=True).stdout.split())
    assert ctypes.sizeof(_RenderConfigC) == size
    assert _RenderConfigC.segmentation.offset == seg_at
    assert seg_at == height_at + 4                # appended after render_height


def test_invalid_segmentation_is_rejected_at_creation(monkeypatch):
    import madrona_b200 as mb
    from madrona_b200.executor import _MaterialViewC, _MeshBVHViewC, _RenderConfigC
    from sims import SIMS, make_executor
    rc = _RenderConfigC(0, _MeshBVHViewC(), _MaterialViewC(), 40, 0.001, 1000.0, 0, 0, 2)
    monkeypatch.setattr(SIMS["gallery"], "render", lambda cfg: (rc, None))
    with pytest.raises(mb.MadronaB200Error, match=r"segmentation = 2 is not 0 \(off\) or 1 \(on\)"):
        make_executor("gallery", 2, num_props=8)


# ---- the C++ facade's overload ---------------------------------------------------------------------------

def _build_facade(tmp_path):
    exe = str(tmp_path / "facade_render_segmentation")
    cmd = ["g++", "-std=c++20", "-O1", "-I" + os.path.join(ROOT, "madrona_b200", "host"),
           os.path.join(ROOT, "tests", "cpp", "facade_render_segmentation.cpp"), "-o", exe,
           "-L" + os.path.join(ROOT, "madrona_b200"), "-lmadrona_b200",
           "-Wl,-rpath," + os.path.join(ROOT, "madrona_b200"),
           "-L/usr/local/cuda/lib64", "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    return exe


def test_facade_segmentation_overload_compiles(tmp_path):
    _build_facade(tmp_path)


@pytest.mark.gpu
def test_gpu_facade_segmentation_overload_matches_python_executor(tmp_path):
    exe = _build_facade(tmp_path)
    assets, out = str(tmp_path / "assets.bin"), str(tmp_path / "frame.bin")
    _write_assets(assets)
    res = subprocess.run([exe, os.path.join(ROOT, "sims", "gallery", "sim.cpp"), assets, out],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    raw = np.fromfile(out, dtype=np.uint8)
    n = 2 * 2 * 64 * 32 * 4
    assert raw.size == 3 * n
    want = _render("gallery", 2, steps=3, width=64, height=32, num_props=40)
    assert np.array_equal(raw[:n], want["rgb"].reshape(-1))
    assert np.array_equal(raw[n:2 * n], want["depth"].reshape(-1).view(np.uint8))
    assert np.array_equal(raw[2 * n:], want["seg"].reshape(-1).view(np.uint8))
    assert (want["seg"] >= 0).mean() > 0.3
