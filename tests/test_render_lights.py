"""Lighting of the batch ray caster (the light loop of renderRaycastKernel, bvh_raycast.cpp:861-919)
and its two prepare kernels: renderLightUpdateKernel (carriers refresh their light entity) and
renderGatherLightsKernel (each world's lights after the light table's world sort).

CPU: the float64 lighting model of tests/lighting_oracle.py against the inline formula of
tests/test_render_bvh.py and against closed-form colours.

GPU, on the gallery_lit fixture (sims/gallery built with -DGALLERY_LIGHTS=1): directional, spot
and point lights with and without shadows, among and above the props, moved and retyped every
step, respawned (lights destroyed and created) every few steps, on two carrier archetypes and one
carrier without a light.  Every clear pixel's colour is checked against the oracle on the lights
as the exported carrier rows describe them at the render: worlds of 0 to 8 lights, flat list and
TLAS, pinhole and panorama, two executors at once, free views, snapshots, and a world past the
8-light cap, which fails the step with ErrRenderLights."""
import glob
import os

import numpy as np
import pytest

from lighting_oracle import GALLERY_LIGHTS, Light, base_colours, engine_normals, shade
from sims.render_assets import GALLERY_MATERIALS, gallery_meshes
from test_render_aspect import camera_rays
from test_render_bvh import _closest_hits, _world_triangles
from test_render_panorama import panorama_rays

FOV_SCALE = 1.0 / np.tan(np.radians(70.0 * 0.5))
OFFSET = np.array([0.0, 0.0, 0.25])     # the gallery cameras' offset
LAMP_SLOTS = {"Lamp": 13, "Beacon": 20}   # position, direction, type, shadow, cutoff, light, world


# ---- CPU: the oracle ---------------------------------------------------------------------------

def _inline_gallery_colour(tris, n, hit_pos, base):
    """the colour formula of tests/test_render_bvh.py for the gallery's two lamps, verbatim"""
    contrib = np.zeros(len(hit_pos))
    ldir = -np.array([0.3, 0.2, -0.9327379])
    facing = (n @ ldir) > 0
    st, _, _ = _closest_hits(hit_pos + 1e-3 * n, np.broadcast_to(ldir, hit_pos.shape), tris, t_min=1e-6)
    lit = facing & ~np.isfinite(st)
    contrib += np.where(lit, np.clip(n @ ldir, 0, 1), 0.0)
    to_l = np.array([0.0, 0.0, 9.0]) - hit_pos
    to_l /= np.linalg.norm(to_l, axis=1, keepdims=True)
    ang = np.arccos(np.clip((-to_l) @ np.array([0.0, 0.0, -1.0]), -1, 1))
    contrib += np.where(np.abs(ang) <= 0.9, np.clip((n * to_l).sum(1), 0, 1), 0.0)
    return np.clip(np.maximum(0.2, contrib)[:, None] * base, 0, 1) * 255.0


def _synthetic_scene(seed):
    """random triangles over a floor: world triangles, and points on them with their normals"""
    rng = np.random.default_rng(seed)
    floor = np.array([[[-10, -10, 0], [10, -10, 0], [10, 10, 0]], [[-10, -10, 0], [10, 10, 0], [-10, 10, 0]]],
                     dtype=np.float64)
    c = rng.uniform([-8, -8, 0.5], [8, 8, 4], size=(40, 3))
    tris = np.concatenate([floor, c[:, None, :] + rng.normal(scale=1.0, size=(40, 3, 3))])
    pick = rng.integers(0, len(tris), size=3000)
    uv = rng.uniform(size=(3000, 2))
    uv = np.where(uv.sum(1, keepdims=True) > 1, 1 - uv, uv)
    a, b, cc = tris[pick, 0], tris[pick, 1], tris[pick, 2]
    hit_pos = a + uv[:, :1] * (b - a) + uv[:, 1:] * (cc - a)
    n = np.cross(b - a, cc - a)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    base = rng.uniform(0.05, 1.0, size=(3000, 3))
    return tris, hit_pos, n, base


def test_oracle_with_the_gallery_lamps_equals_the_inline_formula():
    for seed in range(3):
        tris, hit_pos, n, base = _synthetic_scene(seed)
        got = shade(tris, hit_pos, n, base, GALLERY_LIGHTS)
        want = _inline_gallery_colour(tris, n, hit_pos, base)
        np.testing.assert_allclose(got.value * 255.0, want, rtol=0, atol=1e-9)
        assert np.array_equal(got.rgb, np.floor(want).astype(np.uint8))
        # both lights did something on this scene
        assert got.shadowed.any() and (got.value.max(1) > 0.2 * base.max(1) + 1e-9).any()


def _quad(z=0.0, half=5.0):
    """one upward-facing quad at height z"""
    return np.array([[[-half, -half, z], [half, -half, z], [half, half, z]],
                     [[-half, -half, z], [half, half, z], [-half, half, z]]], dtype=np.float64)


def test_oracle_closed_form_colours_on_one_quad():
    up = np.array([[0.0, 0.0, 1.0]])
    base = np.array([[0.5, 1.0, 0.25]])
    tris = _quad()
    blocker = np.array([[[0.5, -1.0, 3.0], [0.5, 1.0, 3.0], [-1.5, 0.0, 3.0]]])       # above (0, 0)
    beyond = np.array([[[3.5, -1.0, 6.0], [3.5, 1.0, 6.0], [1.5, 0.0, 6.0]]])          # above (2.5, 0)

    def colour(lights, p, scene=tris, n=up):
        s = shade(scene, np.array([p], dtype=np.float64), n, base, lights)
        return s.value[0] / base[0], s

    # a spotlight 4 above the origin pointing down, a 0.5 rad cone: inside at radius 1, outside at 3
    spot = Light(False, False, (0, 0, 4), (0, 0, -1), 0.5)
    k, _ = colour([spot], (1.0, 0.0, 0.0))
    assert np.allclose(k, 4 / np.sqrt(17))                         # n . l, l towards the light
    k, _ = colour([spot], (3.0, 0.0, 0.0))
    assert np.allclose(k, 0.2)                                     # outside: the 0.2 floor
    # the same cone as a point light (cutoff -1): lit everywhere the surface faces it
    point = Light(False, False, (0, 0, 4), (0, 0, -1), -1.0)
    k, _ = colour([point], (3.0, 0.0, 0.0))
    assert np.allclose(k, 4 / 5)
    # a directional light at 60 degrees from the normal
    sun = Light(True, True, (0, 0, 0), (0, -np.sin(np.pi / 3), -np.cos(np.pi / 3)), 0.9)
    k, _ = colour([sun], (0.0, 0.0, 0.0))
    assert np.allclose(k, 0.5)
    # shadowed and unshadowed points of a shadow-casting point light
    point_sh = Light(False, True, (0, 0, 4), (0, 0, -1), -1.0)
    scene = np.concatenate([tris, blocker])
    k, s = colour([point_sh], (0.0, 0.0, 0.0), scene)
    assert np.allclose(k, 0.2) and s.shadowed[0] and not s.beyond[0]
    k, s = colour([point_sh], (0.0, 4.0, 0.0), scene)
    assert np.allclose(k, 1 / np.sqrt(2)) and not s.shadowed[0]
    # an occluder beyond the light still shadows (the shadow ray runs to t = 10000)
    low = Light(False, True, (2.5, 0, 2), (0, 0, -1), 0.8)
    k, s = colour([low], (2.5, 0.0, 0.0), np.concatenate([tris, beyond]))
    assert np.allclose(k, 0.2) and s.shadowed[0] and s.beyond[0]
    k, s = colour([Light(False, False, (2.5, 0, 2), (0, 0, -1), 0.8)], (2.5, 0.0, 0.0),
                  np.concatenate([tris, beyond]))
    assert np.allclose(k, 1.0)
    # a back-facing surface: nothing from any light, shadowed or not
    down = -up
    for l in (spot, point, sun, point_sh):
        k, _ = colour([l], (1.0, 0.0, 0.0), n=down)
        assert np.allclose(k, 0.2)
    # intensity and active are ignored
    dim = Light(False, False, (0, 0, 4), (0, 0, -1), 0.5, intensity=0.1, active=False)
    assert np.array_equal(colour([dim], (1.0, 0.0, 0.0))[0], colour([spot], (1.0, 0.0, 0.0))[0])


def test_oracle_clamps_the_sum_and_floors_an_unlit_world():
    up = np.array([[0.0, 0.0, 1.0]])
    base = np.array([[0.9, 0.5, 0.1]])
    overhead = Light(False, False, (0, 0, 4), (0, 0, -1), -1.0)
    s = shade(_quad(), np.zeros((1, 3)), up, base, [overhead] * 3)
    assert np.allclose(s.value[0], np.minimum(1.0, 3 * base[0]))
    assert np.array_equal(s.rgb[0], np.floor(np.minimum(1.0, 3 * base[0]) * 255).astype(np.uint8))
    s = shade(_quad(), np.zeros((1, 3)), up, base, [])
    assert np.allclose(s.value[0], 0.2 * base[0]) and not s.edge.any()


def test_lit_gallery_fixture_compiles(tmp_path, monkeypatch):
    import madrona_b200 as mb
    from sims import SIMS
    desc = SIMS["gallery_lit"]
    monkeypatch.setenv("MADRONA_B200_KERNEL_CACHE_DIR", str(tmp_path))
    monkeypatch.delenv("MADRONA_B200_NO_KERNEL_CACHE", raising=False)
    mb.precompile(mb.CompileConfig(userSources=desc.sources,
                                   userCompileFlags=["-I" + os.path.dirname(desc.sources[0])] +
                                   list(desc.compile_flags)))
    assert len(glob.glob(str(tmp_path / "*.cubin"))) == 1


# ---- GPU: frames of the lit gallery ------------------------------------------------------------

def _executor(W, lamps, lamps_after=None, lamp_period=0, P=40, res=32, **cfg):
    """a gallery_lit executor of res x res images (or cfg's width x height)"""
    from sims import make_executor
    if "width" not in cfg:
        cfg["resolution"] = res
    return make_executor("gallery_lit", W, num_props=P, lamps=lamps, lamps_after=lamps_after,
                         lamp_period=lamp_period, seed=cfg.pop("seed", 5), **cfg)


def _col(ex, slot, dtype, shape):
    return ex.tensor(slot, dtype, shape).cpu().numpy().copy()


def _lamps(ex):
    """both carrier archetypes' rows as exported: a dict of arrays over all their rows"""
    rows = []
    for kind, s in LAMP_SLOTS.items():
        n = ex.exportedNumRows(s)
        rows.append(dict(kind=np.full(n, kind), pos=_col(ex, s, "float32", (n, 3)),
                         dir=_col(ex, s + 1, "float32", (n, 3)), type=_col(ex, s + 2, "uint8", (n,)),
                         shadow=_col(ex, s + 3, "uint8", (n,)), cutoff=_col(ex, s + 4, "float32", (n,)),
                         light=_col(ex, s + 5, "int32", (n, 2)), world=_col(ex, s + 6, "int32", (n,))))
    return {k: np.concatenate([r[k] for r in rows]) for k in rows[0]}


def _lights_of(lamps, w):
    """world w's lights as the carriers describe them (carriers without a light skipped)"""
    sel = np.nonzero((lamps["world"] == w) & (lamps["light"][:, 1] >= 0))[0]
    return [Light(bool(lamps["type"][i]), bool(lamps["shadow"][i]), lamps["pos"][i].astype(np.float64),
                  lamps["dir"][i].astype(np.float64), float(lamps["cutoff"][i])) for i in sel]


def _frame(ex, W, P, width, height):
    """everything the oracle needs from one render of the lit gallery"""
    return dict(W=W, P=P, width=width, height=height,
                pos=_col(ex, 0, "float32", (W, P, 3)), rot=_col(ex, 1, "float32", (W, P, 4)),
                scale=_col(ex, 2, "float32", (W, P, 3)), obj=_col(ex, 3, "int32", (W, P)),
                mat=_col(ex, 4, "int32", (W, P)), color=_col(ex, 5, "uint32", (W, P)),
                vpos=_col(ex, 6, "float32", (W, 2, 3)), vrot=_col(ex, 7, "float32", (W, 2, 4)),
                rgb=_col(ex, 8, "uint8", (2 * W, height, width, 4)),
                depth=_col(ex, 9, "float32", (2 * W, height, width)), lamps=_lamps(ex))


def _render(ex, render, W, P, width, height):
    ex.run(render)
    return _frame(ex, W, P, width, height)


def _views_of(f, w, panorama=False):
    for v in range(2):
        cam = f["vpos"][w, v].astype(np.float64) + OFFSET
        q = f["vrot"][w, v].astype(np.float64)
        q_inv = np.array([q[0], -q[1], -q[2], -q[3]])
        rays = (panorama_rays if panorama else camera_rays)(cam, q_inv, FOV_SCALE, f["width"], f["height"])
        yield 2 * w + v, cam, rays


class Stats:
    def __init__(self):
        self.checked = self.edge = self.beyond = self.shadowed = 0
        self.max_err = 0


def _check_world(f, w, lights, stats, panorama=False, exact_floor=False):
    """every clear pixel of world w's two views against the oracle; returns the worst view's
    fraction of non-edge pixels within +-1"""
    meshes = gallery_meshes()
    P = f["P"]
    idx = np.array([i for i in range(P) if i == 0 or i % 17 != 0])     # the drawn props
    obj_w, rot_w = f["obj"][w, idx], f["rot"][w, idx]
    tris, owner, src = _world_triangles(meshes, f["pos"][w, idx], rot_w, f["scale"][w, idx], obj_w)
    for view, cam, rays in _views_of(f, w, panorama):
        o = np.broadcast_to(cam, rays.shape)
        t, tri, t2 = _closest_hits(o, rays, tris)
        got_d = f["depth"][view].reshape(-1)
        want_hit, got_hit = np.isfinite(t), got_d > 0
        # silhouettes may differ between the watertight fp32 test and float64 Moeller-Trumbore
        assert (want_hit != got_hit).sum() <= max(1, int(0.005 * len(t))), (w, view)
        both = want_hit & got_hit
        np.testing.assert_allclose(got_d[both], t[both], rtol=1e-4, atol=1e-4)
        with np.errstate(invalid="ignore"):
            clear = both & ((t2 - t) > 1e-3 * np.maximum(t, 1.0))
        sel = np.nonzero(clear)[0]
        inst = owner[tri[sel]]
        n = engine_normals(meshes, obj_w, rot_w, inst, src[tri[sel]])
        base = base_colours(meshes, GALLERY_MATERIALS, obj_w, f["mat"][w, idx], f["color"][w, idx], inst)
        hit_pos = o[sel] + t[sel, None] * rays[sel]
        s = shade(tris, hit_pos, n, base, lights)
        got = f["rgb"][view].reshape(-1, 4)[sel, :3].astype(np.int64)
        err = np.abs(got - s.rgb.astype(np.int64)).max(axis=1)
        keep = ~s.edge
        assert (f["rgb"][view][..., 3] == 255).all()
        if keep.any():
            frac = float((err[keep] <= 1).mean())
            assert frac >= 0.999, (w, view, frac, int(keep.sum()), len(lights))
            assert err[keep].max() <= 3, (w, view, int(err[keep].max()), len(lights))
            stats.max_err = max(stats.max_err, int(err[keep].max()))
        if exact_floor:
            # no lights: max(0.2, 0) * base in float32, truncated
            assert not lights
            b32 = _base_f32(obj_w, f["mat"][w, idx], f["color"][w, idx], inst, meshes)
            want = (np.float32(0.2) * b32 * np.float32(255.0)).astype(np.uint8)
            assert np.array_equal(got.astype(np.uint8), want), (w, view)
        stats.checked += int(keep.sum())
        stats.edge += int(s.edge.sum())
        stats.beyond += int((s.beyond & keep).sum())
        stats.shadowed += int((s.shadowed & keep).sum())


def _base_f32(obj, mat, color, inst, meshes):
    """the kernel's base colour in float32 (hexToRgb / the material table)"""
    out = np.ones((len(inst), 3), dtype=np.float32)
    for j, k in enumerate(inst):
        m = int(mat[k])
        if m == -2:
            hx = int(color[k])
            out[j] = np.array([(hx >> 16) & 255, (hx >> 8) & 255, hx & 255], dtype=np.float32) / np.float32(255.0)
            continue
        if m == -1:
            m = meshes[int(obj[k])][2]
        if m >= 0:
            out[j] = GALLERY_MATERIALS[m, :3].astype(np.float32)
    return out


def _check_frame(f, stats, worlds=None, panorama=False):
    for w in (range(f["W"]) if worlds is None else worlds):
        lights = _lights_of(f["lamps"], w)
        _check_world(f, w, lights, stats, panorama, exact_floor=not lights)


def _counts(f):
    return [len(_lights_of(f["lamps"], w)) for w in range(f["W"])]


def _kinds(f):
    """(directional, point, shadow) of every light of the frame"""
    L = f["lamps"]
    live = L["light"][:, 1] >= 0
    return set(zip(L["type"][live].astype(bool), L["cutoff"][live] == -1.0, L["shadow"][live].astype(bool)))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [40, 100], ids=["flat_list_40_props", "tlas_100_props"])
def test_gpu_lit_pixels_match_the_oracle(P):
    # worlds of 0, 1, 2, 5 and 8 lights; the respawn at step 3 takes them to 3, 0, 5, 2 and 8
    # lights and the one at step 6 back: the renders after steps 5 and 7 see both sets
    lamps, after = [0, 1, 2, 5, 8], [3, 0, 5, 2, 8]
    W, res = len(lamps), 32
    ex = _executor(W, lamps, after, lamp_period=3, P=P)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    stats, frames = Stats(), []
    for t in range(1, 8):
        ex.run(step)
        if t in (5, 7):
            frames.append(_render(ex, render, W, P, res, res))
    ex.close()
    assert _counts(frames[0]) == after and _counts(frames[1]) == lamps
    for f in frames:
        _check_frame(f, stats)
    kinds = _kinds(frames[0]) | _kinds(frames[1])
    # directional, spot and point lights, each with and without shadows
    for directional, point in [(True, False), (False, False), (False, True)]:
        for sh in (False, True):
            assert any(k[0] == directional and (directional or k[1] == point) and k[2] == sh for k in kinds), kinds
    assert stats.checked > 5000 and stats.shadowed > 100, vars(stats)


@pytest.mark.gpu
def test_gpu_moving_lamps_relight_the_image():
    W, P, res = 2, 40, 32
    ex = _executor(W, [2, 5], P=P)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    stats = Stats()
    ex.run(step)
    a = _render(ex, render, W, P, res, res)
    ex.run(step)
    b = _render(ex, render, W, P, res, res)
    ex.close()
    # the carriers moved, turned and flipped flags; the pixels they light changed with them
    assert not np.array_equal(a["lamps"]["pos"], b["lamps"]["pos"])
    assert not np.array_equal(a["lamps"]["dir"], b["lamps"]["dir"])
    for w in range(W):
        assert not np.array_equal(a["rgb"][2 * w:2 * w + 2], b["rgb"][2 * w:2 * w + 2]), w
    for f in (a, b):
        _check_frame(f, stats)
    # spot and point lights with an occluder only past them: their shadow rays run on to t = 10000
    assert stats.checked > 2000 and stats.beyond > 20, vars(stats)


@pytest.mark.gpu
def test_gpu_respawned_lamps_match_the_oracle_at_every_render():
    # world 0 goes from 4 lights to none and back, world 1 from none to 3; a respawn every 2 steps
    lamps, after = [4, 0, 6, 3], [0, 3, 2, 3]
    W, P, res = len(lamps), 40, 24
    ex = _executor(W, lamps, after, lamp_period=2, P=P, res=res, seed=11)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    stats, seen = Stats(), []
    for t in range(1, 7):
        ex.run(step)
        f = _render(ex, render, W, P, res, res)
        seen.append(_counts(f))
        _check_frame(f, stats)
    ex.close()
    # respawns at steps 2 and 6 leave `after`, the one at step 4 `lamps`
    assert seen == [lamps, after, after, lamps, lamps, after], seen
    assert stats.checked > 3000


@pytest.mark.gpu
def test_gpu_both_carrier_archetypes_and_a_carrier_without_a_light():
    W, P, res = 1, 40, 32
    ex = _executor(W, [7], P=P)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(2):
        ex.run(step)
    f = _render(ex, render, W, P, res, res)
    ex.close()
    L = f["lamps"]
    beacon = L["kind"] == "Beacon"
    # lamps 1 and 4 of the world are Beacons, and one Beacon carries no light
    assert beacon.sum() == 3 and (~beacon).sum() == 5
    assert (L["light"][beacon, 1] < 0).sum() == 1 and (L["light"][~beacon, 1] >= 0).all()
    stats = Stats()
    _check_frame(f, stats)
    assert stats.checked > 500
    # the Beacons' lights are drawn: without them the oracle disagrees
    f_lamps_only = dict(f, lamps={k: v[~beacon] for k, v in L.items()})
    with pytest.raises(AssertionError):
        _check_frame(f_lamps_only, Stats())


@pytest.mark.gpu
def test_gpu_two_lit_executors_render_their_own_lights():
    P, res = 40, 32
    a = _executor(2, [2, 5], lamp_period=2, P=P, seed=5)
    b = _executor(2, [8, 1], lamp_period=3, P=P, seed=9)
    ga, ra = a.buildLaunchGraphAllTaskGraphs(), a.buildRenderGraph()
    gb, rb = b.buildLaunchGraphAllTaskGraphs(), b.buildRenderGraph()
    for _ in range(3):
        a.run(ga)
        b.run(gb)
    fa, fb = _render(a, ra, 2, P, res, res), _render(b, rb, 2, P, res, res)
    a.close()
    b.close()
    assert _counts(fa) == [2, 5] and _counts(fb) == [8, 1]
    stats = Stats()
    _check_frame(fa, stats)
    _check_frame(fb, stats)
    assert stats.checked > 2000


@pytest.mark.gpu
def test_gpu_lit_panorama_matches_the_oracle():
    W, P, width, height = 2, 100, 64, 16
    ex = _executor(W, [5, 3], [2, 6], lamp_period=2, P=P, panorama=True, width=width, height=height)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(3):
        ex.run(step)
    f = _render(ex, render, W, P, width, height)
    ex.close()
    assert _counts(f) == [2, 6]
    stats = Stats()
    _check_frame(f, stats, panorama=True)
    assert stats.checked > 500 and stats.shadowed > 20, vars(stats)


@pytest.mark.gpu
def test_gpu_free_views_equal_the_lit_render_graph_bytes():
    W, P, width, height = 2, 100, 48, 32
    ex = _executor(W, [5, 2], [1, 4], lamp_period=2, P=P, width=width, height=height)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for t in range(5):
        ex.run(step)
        ex.run(render)
        vpos, vrot = _col(ex, 6, "float32", (W, 2, 3)), _col(ex, 7, "float32", (W, 2, 4))
        views = [(w, vpos[w, v] + OFFSET.astype(np.float32), vrot[w, v], 70.0) for w in range(W) for v in range(2)]
        got = ex.renderFreeViews(views, width, height, rgb=True, depth=True)
        want = _col(ex, 8, "uint8", (2 * W, height, width, 4))
        assert np.array_equal(got["rgb"].cpu().numpy(), want), t
    ex.close()


@pytest.mark.gpu
def test_gpu_restored_snapshot_renders_the_saved_lights():
    W, P, res = 2, 40, 32
    ex = _executor(W, [4, 2], [1, 5], lamp_period=2, P=P)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    ex.run(step)
    before = _render(ex, render, W, P, res, res)
    with ex.snapshot() as snap:
        snap.save()
        for _ in range(2):      # a respawn at step 2
            ex.run(step)
        moved = _render(ex, render, W, P, res, res)
        assert _counts(moved) != _counts(before)
        assert not np.array_equal(moved["rgb"], before["rgb"])
        snap.restore()
        again = _render(ex, render, W, P, res, res)
    ex.close()
    assert np.array_equal(again["rgb"], before["rgb"])
    assert np.array_equal(again["depth"].view(np.uint32), before["depth"].view(np.uint32))


@pytest.mark.gpu
def test_gpu_a_world_past_the_light_cap_fails_the_step():
    import torch
    import madrona_b200 as mb
    W, P, res = 3, 40, 32
    ex = _executor(W, [9, 8, 3], P=P)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    with pytest.raises(mb.MadronaB200Error, match=r"more than 8 render lights in a world \(the first 8 were drawn\)"):
        ex.run(step)
    # the render of that step still draws the other worlds with all their lights
    try:
        ex.run(render)
    except mb.MadronaB200Error as e:
        assert "render lights" in str(e), str(e)
    f = _frame(ex, W, P, res, res)
    ex.close()
    assert _counts(f) == [9, 8, 3]
    stats = Stats()
    _check_frame(f, stats, worlds=[1, 2])
    assert stats.checked > 500
    # a new executor works
    ex = _executor(1, [8], P=P)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    ex.run(step)
    f = _render(ex, render, 1, P, res, res)
    ex.close()
    torch.cuda.synchronize()
    assert (f["depth"] > 0).mean() > 0.3
    _check_frame(f, stats)
