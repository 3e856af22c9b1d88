"""Ray casting worlds of any size: compact per-world instance lists and the global-memory
TLAS builder for worlds above 128 instances (kernels_render.cu).

  * every world's TLAS, on both sides of the 128-instance threshold and after the props
    moved and the tables grew, equals the numpy restatement of the build rules
    (tests/tlas_model.py) byte for byte after depth-first canonicalisation;
  * at 2000 instances per world every pixel follows the brute-force float64 closest hit of
    tests/test_render_bvh.py, with the same thresholds;
  * a clustered world whose tree is too deep for the traversal stack fails `run` with the
    render error instead of rendering with geometry missing;
  * worlds of up to 128 instances write the same bytes as before (stored digests)."""
import json
import os

import numpy as np
import pytest

from tlas_model import MAX_TLAS_DEPTH, build_tlas, canonicalise, same_tree

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _visible(props):
    # the gallery hides every 17th prop (never the ground, prop 0)
    return 0 if props == 0 else props - (props - 1) // 17


def _props_for(visible):
    p = visible
    while _visible(p) < visible:
        p += 1
    assert _visible(p) == visible
    return p


def _make(monkeypatch, props, **cfg):
    from sims import make_executor
    # tables start with room for every prop (the entity store is sized from them, and world
    # construction has to fit it); they are more than half full, so they double after the
    # first step and the instance list grows with them
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", str(-(-sum(props) // len(props)) + 64))
    return make_executor("gallery_sized", len(props), props=props, **cfg)


def _instance_boxes(inst_raw):
    f = inst_raw.copy().view(np.float32).reshape(-1, 19)
    return f[:, 13:16], f[:, 16:19]


@pytest.mark.gpu
def test_gpu_tlas_matches_model_across_sizes_and_growth(monkeypatch):
    sizes = [0, 1, 40, 128, 129, 513, 2000, 9000]
    ex = _make(monkeypatch, [_props_for(v) for v in sizes], seed=11, resolution=16, rgbd=True)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    prev = None
    for s in range(4):
        ex.run(step)
        nodes, ncount, inst, icount, offsets = ex.renderDebugStructures()
        assert icount.tolist() == sizes
        assert offsets.tolist() == np.concatenate([[0], np.cumsum(sizes)[:-1]]).tolist()
        lo, hi = _instance_boxes(inst)
        for w, n in enumerate(sizes):
            o = int(offsets[w])
            want, depth = build_tlas(lo[o:o + n], hi[o:o + n])
            assert int(ncount[w]) == len(want) and len(want) <= max(1, n - 1)
            got = canonicalise(nodes[o:o + int(ncount[w])])
            assert same_tree(got, want), (s, w, n)
            assert depth <= MAX_TLAS_DEPTH
        if prev is not None:
            assert not np.array_equal(prev, lo)          # the props moved: new trees
        prev = lo.copy()
    ex.run(render)
    ex.close()


# ---- pixels against the brute-force closest hit ------------------------------------------------

def _check_pixels(ex, props, res):
    """tests/test_render_bvh.py's per-pixel pin for worlds of different sizes."""
    import madrona_b200 as mb
    from sims.render_assets import GALLERY_MATERIALS, gallery_meshes
    from test_render_bvh import _camera_rays, _closest_hits, _world_triangles

    W = len(props)
    rows = int(sum(props))
    assert ex.exportedNumRows(0) == rows and ex.exportedNumRows(8) == 2 * W

    def col(slot, dtype, shape):
        return ex.tensor(slot, dtype, shape).cpu().numpy()
    pos, rot = col(0, "float32", (rows, 3)), col(1, "float32", (rows, 4))
    scale, obj = col(2, "float32", (rows, 3)), col(3, "int32", (rows,))
    mat, color = col(4, "int32", (rows,)), col(5, "uint32", (rows,))
    vpos, vrot = col(6, "float32", (W, 2, 3)), col(7, "float32", (W, 2, 4))
    rgb = col(8, "uint8", (2 * W, res, res, 4))
    depth = col(9, "float32", (2 * W, res, res))
    hits = ex.renderDebugHits(2 * W, res).cpu().numpy()

    meshes = gallery_meshes()
    bvh = mb.MeshBVHData(meshes, gpu_id=-1)
    src_of = bvh.triangle_sources()
    first_tri = np.cumsum([0] + [len(m[1]) for m in meshes])
    fov_scale = 1.0 / np.tan(np.radians(70.0 * 0.5))

    total, id_checked, rgb_checked = 0, 0, 0
    start = 0
    for w, P in enumerate(props):
        rows_w = slice(start, start + P)
        start += P
        visible = np.array([i == 0 or i % 17 != 0 for i in range(P)])
        idx = np.nonzero(visible)[0]              # instance k of the engine = k-th visible prop
        wp, wr, ws, wo = pos[rows_w][idx], rot[rows_w][idx], scale[rows_w][idx], obj[rows_w][idx]
        wm, wc = mat[rows_w][idx], color[rows_w][idx]
        tris, owner, src = _world_triangles(meshes, wp, wr, ws, wo)
        for v in range(2):
            view = 2 * w + v
            cam = vpos[w, v].astype(np.float64) + np.array([0.0, 0.0, 0.25])
            q = vrot[w, v].astype(np.float64)
            rays = _camera_rays(cam, np.array([q[0], -q[1], -q[2], -q[3]]), fov_scale, res)
            o = np.broadcast_to(cam, rays.shape)
            t, tri, t2 = _closest_hits(o, rays, tris)
            want_hit = np.isfinite(t)
            got_d = depth[view].reshape(-1)
            got_hit = got_d > 0
            total += len(t)
            assert (want_hit == got_hit).mean() > 0.995
            both = want_hit & got_hit
            np.testing.assert_allclose(got_d[both], t[both], rtol=1e-4, atol=1e-4)
            with np.errstate(invalid="ignore"):
                clear = both & ((t2 - t) > 1e-3 * np.maximum(t, 1.0))
            g_inst, g_tri = hits[view].reshape(-1, 2)[:, 0], hits[view].reshape(-1, 2)[:, 1]
            want_inst = owner[np.maximum(tri, 0)]
            assert np.array_equal(g_inst[clear], want_inst[clear])
            got_src = src_of[first_tri[wo[want_inst]] + np.maximum(g_tri, 0)]
            assert np.array_equal(got_src[clear], src[np.maximum(tri, 0)][clear])
            id_checked += int(clear.sum())

            sel = np.nonzero(clear)[0]
            inst_k = want_inst[sel]
            n_obj = []
            for k, s_tri in zip(inst_k, src[tri[sel]]):
                vtx, f, _ = meshes[int(wo[k])]
                a, b, c = vtx[f[s_tri]].astype(np.float64)
                nn = np.cross(b - a, c - a)
                nn = nn / np.linalg.norm(nn)
                u = wr[k].astype(np.float64)
                uv = np.array(u[1:])
                n_obj.append(nn + 2.0 * np.cross(uv, np.cross(uv, nn) + u[0] * nn))
            n = np.array(n_obj).reshape(-1, 3)
            hit_pos = o[sel] + t[sel, None] * rays[sel]
            contrib = np.zeros(len(sel))
            ldir = -np.array([0.3, 0.2, -0.9327379])
            facing = (n @ ldir) > 0
            st, _, _ = _closest_hits(hit_pos + 1e-3 * n, np.broadcast_to(ldir, hit_pos.shape), tris, t_min=1e-6)
            lit = facing & ~np.isfinite(st)
            st_a, _, _ = _closest_hits(hit_pos + 3e-3 * n, np.broadcast_to(ldir, hit_pos.shape), tris, t_min=1e-6)
            st_b, _, _ = _closest_hits(hit_pos + 3e-4 * n, np.broadcast_to(ldir, hit_pos.shape), tris, t_min=1e-6)
            graze = (np.isfinite(st) != np.isfinite(st_a)) | (np.isfinite(st) != np.isfinite(st_b))
            contrib += np.where(lit, np.clip(n @ ldir, 0, 1), 0.0)
            to_l = np.array([0.0, 0.0, 9.0]) - hit_pos
            to_l /= np.linalg.norm(to_l, axis=1, keepdims=True)
            ang = np.arccos(np.clip((-to_l) @ np.array([0.0, 0.0, -1.0]), -1, 1))
            contrib += np.where(np.abs(ang) <= 0.9, np.clip((n * to_l).sum(1), 0, 1), 0.0)
            base = np.ones((len(sel), 3))
            for j, k in enumerate(inst_k):
                m = int(wm[k])
                if m == -2:
                    hx = int(wc[k])
                    base[j] = [((hx >> 16) & 255) / 255.0, ((hx >> 8) & 255) / 255.0, (hx & 255) / 255.0]
                else:
                    if m == -1:
                        m = meshes[int(wo[k])][2]
                    if m >= 0:
                        base[j] = GALLERY_MATERIALS[m, :3]
            want_rgb = np.clip(np.maximum(0.2, contrib)[:, None] * base, 0, 1) * 255.0
            got_rgb = rgb[view].reshape(-1, 4)[sel, :3].astype(np.float64)
            edge = graze | (np.abs(np.abs(ang) - 0.9) < 5e-3) | (np.abs(n @ ldir) < 5e-3)
            ok = np.abs(got_rgb - want_rgb).max(axis=1) <= 2.0
            assert ok[~edge].mean() > 0.99, (w, v, float(ok[~edge].mean()), float(edge.mean()))
            assert (rgb[view][..., 3] == 255).all()
            rgb_checked += int((~edge).sum())
    return total, id_checked, rgb_checked


@pytest.mark.gpu
def test_gpu_hits_match_brute_force_closest_hit_at_2000_instances(monkeypatch):
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    props, res = [_props_for(2001)], 24
    ex = _make(monkeypatch, props, seed=5, resolution=res, rgbd=True)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(2):
        ex.run(step)
    ex.run(render)
    total, id_checked, rgb_checked = _check_pixels(ex, props, res)
    ex.close()
    assert id_checked > 0.8 * total * 0.5 and rgb_checked > 500


@pytest.mark.gpu
def test_gpu_clustered_world_renders_whole_or_fails_with_the_render_error(monkeypatch):
    import madrona_b200 as mb

    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    # world 0: clustered, 300 props (large builder); world 1: scattered, 200 props
    props, res = [300, 200], 24
    ex = _make(monkeypatch, props, layouts=[1, 0], seed=7, resolution=res, rgbd=True)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    failure = None
    try:
        ex.run(step)
    except mb.MadronaB200Error as e:
        failure = str(e)
    nodes, ncount, inst, icount, offsets = ex.renderDebugStructures()
    lo, hi = _instance_boxes(inst)
    depths = [build_tlas(lo[o:o + n], hi[o:o + n])[1] for o, n in zip(offsets.tolist(), icount.tolist())]
    if max(depths) > MAX_TLAS_DEPTH:
        assert failure is not None and "TLAS too deep" in failure, failure
    else:
        assert failure is None, failure
        ex.run(render)
        _check_pixels(ex, props, res)
    assert depths[0] > MAX_TLAS_DEPTH      # the layout exists to make a deep tree
    ex.close()


@pytest.mark.gpu
def test_gpu_small_worlds_write_the_same_images_as_before():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_render_digests",
                                                  os.path.join(GOLDEN, "make_render_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    with open(os.path.join(GOLDEN, "render_digests.json")) as f:
        want = json.load(f)
    assert mod.render_digests() == want
