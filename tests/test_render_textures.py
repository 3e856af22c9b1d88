"""Material textures in the batch ray caster (bvh_raycast.cpp:788-800) and their upload
(mb2_init_material_data, role of render::AssetProcessor::initMaterialData).

CPU: a numpy model of the texture unit's linear filter, a BC7 mode-6 encoder / decoder,
and the upload's input checks (which run before any CUDA call).  GPU: textured colour
against a brute-force float64 closest hit whose barycentrics interpolate the uvs and
whose texel lookup goes through the filter model; textures must change colour only."""
import numpy as np
import pytest

from sims.render_assets import (bc7_mode6_decode, bc7_mode6_encode, gallery_textured_materials,
                                gallery_textured_meshes, gallery_textures)


# ---- linear filtering model ---------------------------------------------------------------------
# CUDA C++ Programming Guide, "Texture Fetching" / "Linear Filtering", normalized coordinates with
# cudaAddressModeWrap: x = frac(u) * W - 0.5, i = floor(x), alpha = frac(x) kept in 9-bit fixed
# point with 8 fractional bits; texels are unorm8 / 255; neighbours wrap.

def tex2d_linear(texels, u, v):
    """texels uint8 [H, W, C]; u, v arrays of normalized coordinates -> float64 [..., C]."""
    H, W = texels.shape[:2]
    u = np.asarray(u, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    x = (u - np.floor(u)) * W - 0.5
    y = (v - np.floor(v)) * H - 0.5
    i, j = np.floor(x), np.floor(y)
    a = np.round((x - i) * 256.0) / 256.0
    b = np.round((y - j) * 256.0) / 256.0
    i0, j0 = i.astype(np.int64) % W, j.astype(np.int64) % H
    i1, j1 = (i0 + 1) % W, (j0 + 1) % H
    T = texels.astype(np.float64) / 255.0
    a, b = a[..., None], b[..., None]
    return ((1 - a) * (1 - b) * T[j0, i0] + a * (1 - b) * T[j0, i1] +
            (1 - a) * b * T[j1, i0] + a * b * T[j1, i1])


def _distinct_texels(H, W):
    j, i = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    return np.stack([17 * i + 3, 29 * j + 5, 7 * (i + j), np.full(i.shape, 255)], -1).astype(np.uint8)


def test_filter_model_is_exact_at_texel_centres_of_a_non_square_texture():
    tex = _distinct_texels(2, 5)                       # 5 wide, 2 high
    j, i = np.meshgrid(np.arange(2), np.arange(5), indexing="ij")
    got = tex2d_linear(tex, (i + 0.5) / 5, (j + 0.5) / 2)
    np.testing.assert_allclose(got, tex / 255.0, atol=1e-12)
    # the same centres one and three periods away
    np.testing.assert_allclose(tex2d_linear(tex, (i + 0.5) / 5 + 1, (j + 0.5) / 2 - 3), tex / 255.0, atol=1e-12)


def test_filter_model_wraps_at_both_seams():
    tex = _distinct_texels(4, 8)
    T = tex / 255.0
    # u = 0: halfway between the last and the first column; v = 0 likewise for rows
    np.testing.assert_allclose(tex2d_linear(tex, 0.0, 0.5 / 4), 0.5 * (T[0, 7] + T[0, 0]), atol=1e-12)
    np.testing.assert_allclose(tex2d_linear(tex, 0.5 / 8, 0.0), 0.5 * (T[3, 0] + T[0, 0]), atol=1e-12)
    corner = 0.25 * (T[3, 7] + T[3, 0] + T[0, 7] + T[0, 0])
    for u, v in ((0.0, 0.0), (1.0, 1.0), (-2.0, 3.0)):
        np.testing.assert_allclose(tex2d_linear(tex, u, v), corner, atol=1e-12)
    # negative coordinates wrap to the same place as their positive twins
    np.testing.assert_allclose(tex2d_linear(tex, -0.3, -0.7), tex2d_linear(tex, 0.7, 0.3), atol=1e-12)


def test_filter_model_weights_have_eight_fractional_bits():
    tex = np.zeros((1, 2, 4), dtype=np.uint8)
    tex[0, 1] = 255
    # x = u * 2 - 0.5 = 1/3 past texel 0: alpha = round(256 / 3) / 256 = 85 / 256
    got = tex2d_linear(tex, (0.5 + 1.0 / 3.0) / 2.0, 0.5)
    assert got[0] == pytest.approx(85 / 256, abs=1e-12)


# ---- BC7 mode 6 -----------------------------------------------------------------------------------

def _block_bits(c, p, idx):
    """Mode-6 block from 7-bit endpoints c[2][4], p-bits p[2] and 16 indices (bit by bit)."""
    bits, pos = 1 << 6, 7
    for ch in range(4):
        for e in range(2):
            bits |= c[e][ch] << pos
            pos += 7
    bits |= p[0] << pos
    bits |= p[1] << (pos + 1)
    pos += 2
    for k in range(16):
        bits |= idx[k] << pos
        pos += 3 if k == 0 else 4
    return np.frombuffer(bits.to_bytes(16, "little"), dtype=np.uint8).reshape(1, 1, 16)


def test_bc7_decoder_follows_the_mode6_layout():
    c = [[10, 100, 0, 127], [90, 20, 127, 127]]
    idx = [0, 15, 7, 8] + [3] * 12
    out = bc7_mode6_decode(_block_bits(c, [1, 0], idx))
    e0 = np.array([21, 201, 1, 255])          # (c << 1) | p
    e1 = np.array([180, 40, 254, 254])
    w = np.array([0, 4, 9, 13, 17, 21, 26, 30, 34, 38, 43, 47, 51, 55, 60, 64])
    want = ((64 - w[:, None]) * e0 + w[:, None] * e1 + 32) >> 6
    assert np.array_equal(out.reshape(16, 4), want[idx])


def test_bc7_round_trip():
    # constant blocks come back exactly when their channels share a parity (one p-bit per
    # endpoint), within 1 otherwise
    flat = np.zeros((8, 8, 4), dtype=np.uint8)
    flat[:4, :4], flat[:4, 4:], flat[4:, :4], flat[4:, 4:] = (0, 0, 0, 0), (255, 255, 255, 255), \
        (17, 201, 3, 255), (128, 2, 254, 90)
    enc = bc7_mode6_encode(flat)
    assert enc.shape == (2, 2, 16) and (enc[..., 0] & 0x7F == 0x40).all()
    assert np.array_equal(bc7_mode6_decode(enc), flat)
    mixed = np.broadcast_to(np.array([128, 1, 254, 91], dtype=np.uint8), (4, 4, 4))
    assert np.abs(bc7_mode6_decode(bc7_mode6_encode(mixed)).astype(int) - mixed).max() <= 1
    # smooth ramps (all channels along one line per block) within a few units
    x, y = np.meshgrid(np.arange(32), np.arange(16))
    t = (x + 2 * y) / 63.0
    ramp = np.stack([255 * t, 255 * (1 - t), 64 + 100 * t, np.full(t.shape, 255)], -1).round().astype(np.uint8)
    dec = bc7_mode6_decode(bc7_mode6_encode(ramp))
    assert np.abs(dec.astype(int) - ramp).max() <= 4
    # blocks whose first texel is nearer the high end need the endpoint swap (3-bit anchor index)
    swap = np.zeros((4, 4, 4), dtype=np.uint8)
    swap[..., 3] = 255
    swap[0, 0, :3] = 250
    swap[3, 3, :3] = 4
    for block in (swap, swap[::-1, ::-1]):
        assert np.abs(bc7_mode6_decode(bc7_mode6_encode(block)).astype(int) - block).max() <= 4


# ---- upload: input checks (no GPU needed: they run before the first CUDA call) -------------------

def _upload(materials, textures):
    import madrona_b200 as mb
    return mb.MaterialData(materials, textures, gpu_id=0)


_MAT = [((1.0, 1.0, 1.0, 1.0), -1, 0.5, 0.0)]
_RGBA = (bytes(4 * 4 * 2), 0, 4, 2)


@pytest.mark.parametrize("materials,textures,message", [
    (_MAT, [(bytes(32), 2, 4, 2)], "unknown format 2"),
    (_MAT, [(bytes(0), 0, 0, 2)], "zero width or height"),
    (_MAT, [(bytes(0), 0, 4, 0)], "zero width or height"),
    (_MAT, [(None, 0, 4, 2)], "no pixel data"),
    (_MAT, [(bytes(31), 0, 4, 2)], "num_bytes is 31, 4 x 2 RGBA8 needs 32"),
    (_MAT, [(bytes(64), 1, 8, 6)], "BC7 width and height must be multiples of 4"),
    (_MAT, [(bytes(6 * 4), 1, 6, 4)], "BC7 width and height must be multiples of 4"),
    (_MAT, [(bytes(16), 1, 8, 4)], "num_bytes is 16, 8 x 4 BC7 needs 32"),
    ([((1, 1, 1, 1), 1, 0.5, 0.0)], [_RGBA], "material 0: texture_idx 1 is outside [-1, 1)"),
    ([_MAT[0], ((1, 1, 1, 1), -2, 0.5, 0.0)], [_RGBA], "material 1: texture_idx -2 is outside [-1, 1)"),
    ([((1, 1, 1, 1), 0, 0.5, 0.0)], [], "material 0: texture_idx 0 is outside [-1, 0)"),
    ([], [_RGBA], "no materials"),
], ids=["format", "zero_width", "zero_height", "null_pixels", "rgba_bytes", "bc7_height", "bc7_width",
        "bc7_bytes", "index_past_end", "index_below_minus_one", "index_without_textures", "no_materials"])
def test_material_upload_rejects_bad_input_before_cuda(materials, textures, message):
    import madrona_b200 as mb
    with pytest.raises(mb.MadronaB200Error, match="mb2_init_material_data: .*" + message.replace("[", r"\[")
                       .replace("(", r"\(").replace(")", r"\)")):
        _upload(materials, textures)


def test_material_upload_needs_a_device_id():
    import madrona_b200 as mb
    with pytest.raises(mb.MadronaB200Error, match="gpu_id must name a device"):
        mb.MaterialData(_MAT, [_RGBA], gpu_id=-1)


def test_textured_gallery_keeps_the_gallery_geometry():
    from sims.render_assets import gallery_meshes
    for (v, f, m), (tv, tf, tm, uv) in zip(gallery_meshes(), gallery_textured_meshes()):
        assert np.array_equal(v, tv) and np.array_equal(f, tf) and m == tm
        assert uv.shape == (len(v), 2) and uv.dtype == np.float32
    assert gallery_textured_meshes()[4][3].max() == 6.0
    assert sum(m[1] >= 0 for m in gallery_textured_materials()) == 2
    shapes = [t.shape for t, _, _ in gallery_textures()]
    assert shapes == [(8, 8, 4), (32, 64, 4), (16, 16, 4)]


# ---- GPU ----------------------------------------------------------------------------------------

def _quat_rotate(q, v):
    w, x, y, z = q
    u = np.array([x, y, z], dtype=np.float64)
    return v + 2.0 * np.cross(u, np.cross(u, v) + w * v)


def _rot_matrix(q):
    return np.stack([_quat_rotate(q, e) for e in np.eye(3)], axis=1)


def _world_triangles(meshes, pos, rot, scale, obj):
    """All triangles of a world: [T, 3, 3] float64, their uvs [T, 3, 2], owner instance [T],
    source triangle [T]."""
    tris, uvs, inst, src = [], [], [], []
    for i in range(len(pos)):
        v, f, _, uv = meshes[int(obj[i])]
        M = _rot_matrix(rot[i].astype(np.float64)) * scale[i].astype(np.float64)[None, :]
        wv = v.astype(np.float64) @ M.T + pos[i].astype(np.float64)
        tris.append(wv[f])
        uvs.append(uv.astype(np.float64)[f])
        inst.append(np.full(len(f), i))
        src.append(np.arange(len(f)))
    return np.concatenate(tris), np.concatenate(uvs), np.concatenate(inst), np.concatenate(src)


def _closest_hits(o, d, tris, t_min=0.0, chunk=256):
    """Moeller-Trumbore in float64 -> (t, tri, second-best t, barycentrics (b1, b2) of the hit)."""
    R = len(d)
    best = np.full(R, np.inf)
    second = np.full(R, np.inf)
    best_tri = np.full(R, -1)
    bary = np.zeros((R, 2))
    e1 = tris[:, 1] - tris[:, 0]
    e2 = tris[:, 2] - tris[:, 0]
    for s in range(0, len(tris), chunk):
        a, b, c = tris[s:s + chunk, 0], e1[s:s + chunk], e2[s:s + chunk]
        p = np.cross(d[:, None, :], c[None, :, :])
        det = (b[None] * p).sum(-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / det
            tv = o[:, None, :] - a[None]
            u = (tv * p).sum(-1) * inv
            q = np.cross(tv, b[None])
            v = (d[:, None, :] * q).sum(-1) * inv
            t = (c[None] * q).sum(-1) * inv
        ok = (np.abs(det) > 1e-14) & (u >= 0) & (v >= 0) & (u + v <= 1) & (t > t_min)
        t = np.where(ok, t, np.inf)
        order = np.sort(t, axis=1)
        cand = t.argmin(axis=1)
        rows = np.arange(R)
        cand_t = t[rows, cand]
        second_here = order[:, 1] if t.shape[1] > 1 else np.full(R, np.inf)
        new_best = cand_t < best
        second = np.where(new_best, np.minimum(best, second_here), np.minimum(second, cand_t))
        best_tri = np.where(new_best, s + cand, best_tri)
        bary = np.where(new_best[:, None], np.stack([u[rows, cand], v[rows, cand]], 1), bary)
        best = np.where(new_best, cand_t, best)
    return best, best_tri, second, bary


def _camera_rays(pos, rot_inv, fov_scale, res):
    """bvh_raycast.cpp:58-88 in float64."""
    q_inv = rot_inv.astype(np.float64)
    q = np.array([q_inv[0], -q_inv[1], -q_inv[2], -q_inv[3]])
    fwd = _quat_rotate(q, np.array([0.0, 1.0, 0.0]))
    fwd /= np.linalg.norm(fwd)
    u = _quat_rotate(q, np.array([1.0, 0.0, 0.0]))
    h = 1.0 / fov_scale
    vv = np.cross(fwd, u)
    vv /= np.linalg.norm(vv)
    horizontal, vertical = u * 2 * h, vv * 2 * h
    ll = pos - horizontal / 2 - vertical / 2 + fwd
    px = (np.arange(res) + 0.5) / res
    d = ll[None, None] + px[None, :, None] * horizontal + px[:, None, None] * vertical - pos
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return d.reshape(-1, 3)


def _render(name, W, P, res, rgbd=True, seed=5, **cfg):
    """Run 3 steps + one render; returns the exported columns and the debug hit ids."""
    from sims import make_executor
    ex = make_executor(name, W, num_props=P, seed=seed, resolution=res, rgbd=rgbd, **cfg)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(3):
        ex.run(step)
    ex.run(render)

    def col(slot, dtype, shape):
        return ex.tensor(slot, dtype, shape).cpu().numpy()
    out = dict(pos=col(0, "float32", (W, P, 3)), rot=col(1, "float32", (W, P, 4)),
               scale=col(2, "float32", (W, P, 3)), obj=col(3, "int32", (W, P)),
               mat=col(4, "int32", (W, P)), color=col(5, "uint32", (W, P)),
               vpos=col(6, "float32", (W, 2, 3)), vrot=col(7, "float32", (W, 2, 4)),
               depth=col(9, "float32", (2 * W, res, res)),
               hits=ex.renderDebugHits(2 * W, res).cpu().numpy())
    if rgbd:
        out["rgb"] = col(8, "uint8", (2 * W, res, res, 4))
    ex.close()
    return out


def _check_textured_colour(r, W, P, res, bc7, cover):
    """Every clear, non-edge pixel against the float64 oracle; counts what was covered."""
    meshes = gallery_textured_meshes()
    materials = gallery_textured_materials(bc7)
    texels = [t for t, _, _ in gallery_textures()]
    fov_scale = 1.0 / np.tan(np.radians(70.0 * 0.5))
    checked = 0
    for w in range(W):
        idx = np.array([i for i in range(P) if i == 0 or i % 17 != 0])      # the visible props
        obj_w, mat_w, col_w = r["obj"][w, idx], r["mat"][w, idx], r["color"][w, idx]
        tris, tri_uv, owner, src = _world_triangles(meshes, r["pos"][w, idx], r["rot"][w, idx],
                                                    r["scale"][w, idx], obj_w)
        for v in range(2):
            view = 2 * w + v
            cam = r["vpos"][w, v].astype(np.float64) + np.array([0.0, 0.0, 0.25])
            q = r["vrot"][w, v].astype(np.float64)
            rays = _camera_rays(cam, np.array([q[0], -q[1], -q[2], -q[3]]), fov_scale, res)
            o = np.broadcast_to(cam, rays.shape)
            t, tri, t2, bary = _closest_hits(o, rays, tris)
            got_d = r["depth"][view].reshape(-1)
            both = np.isfinite(t) & (got_d > 0)
            with np.errstate(invalid="ignore"):
                clear = both & ((t2 - t) > 1e-3 * np.maximum(t, 1.0))
            want_inst = owner[np.maximum(tri, 0)]
            g_inst = r["hits"][view].reshape(-1, 2)[:, 0]
            clear &= g_inst == want_inst
            sel = np.nonzero(clear)[0]
            inst_k = want_inst[sel]

            # uv of the float64 hit: (1 - b1 - b2) uv_a + b1 uv_b + b2 uv_c
            b1, b2 = bary[sel, 0], bary[sel, 1]
            tuv = tri_uv[tri[sel]]
            uv = (1 - b1 - b2)[:, None] * tuv[:, 0] + b1[:, None] * tuv[:, 1] + b2[:, None] * tuv[:, 2]

            # lighting restated from bvh_raycast.cpp:848-938 (see tests/test_render_bvh.py)
            n_obj = []
            for k, s_tri in zip(inst_k, src[tri[sel]]):
                vtx, f, _, _ = meshes[int(obj_w[k])]
                a, b, c = vtx[f[s_tri]].astype(np.float64)
                nn = np.cross(b - a, c - a)
                n_obj.append(_quat_rotate(r["rot"][w, idx][k].astype(np.float64), nn / np.linalg.norm(nn)))
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

            # base colour: override colour, else material colour x filtered texel at (u, 1 - v)
            base = np.ones((len(sel), 3))
            tex_of = np.full(len(sel), -1)
            for j, k in enumerate(inst_k):
                m = int(mat_w[k])
                if m == -2:
                    hx = int(col_w[k])
                    base[j] = [((hx >> 16) & 255) / 255.0, ((hx >> 8) & 255) / 255.0, (hx & 255) / 255.0]
                    continue
                if m == -1:
                    m = meshes[int(obj_w[k])][2]
                if m >= 0:
                    color, ti = materials[m][0], materials[m][1]
                    base[j] = color[:3]
                    if ti >= 0:
                        tex_of[j] = ti
                        base[j] *= tex2d_linear(texels[ti], uv[j, 0], 1.0 - uv[j, 1])[:3]
            want_rgb = np.clip(np.maximum(0.2, contrib)[:, None] * base, 0, 1) * 255.0
            got_rgb = r["rgb"][view].reshape(-1, 4)[sel, :3].astype(np.float64)
            edge = graze | (np.abs(np.abs(ang) - 0.9) < 5e-3) | (np.abs(n @ ldir) < 5e-3)
            ok = np.abs(got_rgb - want_rgb).max(axis=1) <= 2.0
            assert ok[~edge].mean() >= 0.99, (w, v, float(ok[~edge].mean()), int((~edge).sum()))
            keep = ~edge & ok
            m_inst = mat_w[inst_k]
            for ti in range(3):
                cover[f"texture_{ti}"] += int((keep & (tex_of == ti)).sum())
            cover["override_textured"] += int((keep & (m_inst >= 0) & (tex_of >= 0)).sum())
            cover["override_colour"] += int((keep & (m_inst == -2)).sum())
            wrapped = (uv < 0).any(1) | (uv >= 1).any(1)
            cover["ground_wrapped"] += int((keep & (obj_w[inst_k] == 4) & wrapped & (tex_of >= 0)).sum())
            checked += int((~edge).sum())
    return checked


@pytest.mark.gpu
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_instances", "flat_list_40_instances"])
def test_gpu_textured_colour_matches_brute_force_oracle(monkeypatch, P):
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    W, res = 3, 40
    cover = {k: 0 for k in ("texture_0", "texture_1", "texture_2", "override_textured", "override_colour",
                            "ground_wrapped")}
    checked = 0
    for bc7 in (False, True):
        r = _render("gallery_textured", W, P, res, bc7=bc7)
        checked += _check_textured_colour(r, W, P, res, bc7, cover)
    assert checked > 1000
    assert all(v > 0 for v in cover.values()), cover


@pytest.mark.gpu
@pytest.mark.parametrize("P", [100, 40], ids=["tlas_100_instances", "flat_list_40_instances"])
def test_gpu_textures_change_colour_only(monkeypatch, P):
    monkeypatch.setenv("MADRONA_B200_RENDER_DEBUG", "1")
    W, res = 2, 40
    plain = _render("gallery", W, P, res)
    textured = _render("gallery_textured", W, P, res)
    assert np.array_equal(plain["depth"].view(np.uint32), textured["depth"].view(np.uint32))
    assert np.array_equal(plain["hits"], textured["hits"])
    assert (plain["depth"] > 0).mean() > 0.3
    # the colours do differ where a textured material was hit
    assert (plain["rgb"] != textured["rgb"]).any()
    # depth-only mode with textured materials writes the same depth
    depth_only = _render("gallery_textured", W, P, res, rgbd=False)
    assert np.array_equal(depth_only["depth"].view(np.uint32), textured["depth"].view(np.uint32))
    assert np.array_equal(depth_only["hits"], textured["hits"])


@pytest.mark.gpu
def test_gpu_texture_index_past_the_config_fails_the_render(monkeypatch):
    """Materials made without mb2_init_material_data carry no texture count: a textureIdx past
    materialData.numTextureBuffers is caught on the device and fails run() with a message."""
    import torch
    import madrona_b200 as mb
    from madrona_b200.executor import _MaterialViewC, _RenderConfigC
    from sims import SIMS, make_executor

    def render_cfg(cfg):
        gpu = int(cfg.get("_gpu_id", 0))
        bvh = mb.MeshBVHData(gallery_textured_meshes(), gpu_id=gpu)
        tex = [(src, fmt, t.shape[1], t.shape[0]) for t, fmt, src in gallery_textures()]
        mats = mb.MaterialData(gallery_textured_materials(), tex, gpu_id=gpu)
        raw = np.zeros((4, 7), dtype=np.float32)
        raw[:, :4] = 1.0
        raw[:, 4] = np.array([3, -1, -1, -1], dtype=np.int32).view(np.float32)   # 3 textures exist
        dev = torch.from_numpy(raw).to(f"cuda:{gpu}")
        view = mats.view()
        mv = _MaterialViewC(view.textures, view.num_texture_buffers, view.texture_buffers, dev.data_ptr())
        return _RenderConfigC(0, bvh.view(device=True), mv, 24, 0.001, 1000.0), [bvh, mats, dev]

    monkeypatch.setattr(SIMS["gallery_textured"], "render", render_cfg)
    ex = make_executor("gallery_textured", 2, num_props=20, seed=1)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    ex.run(step)
    with pytest.raises(mb.MadronaB200Error, match="render asset error"):
        ex.run(render)
    ex.close()


@pytest.mark.gpu
def test_gpu_material_data_lifetime():
    """The executor adopts the handle's pointers: executors are destroyed first, then the
    handle; one handle can serve two executors at once."""
    import madrona_b200 as mb
    from madrona_b200.executor import _RenderConfigC
    from sims import SIMS, make_executor

    bvh = mb.MeshBVHData(gallery_textured_meshes(), gpu_id=0)
    tex = [(src, fmt, t.shape[1], t.shape[0]) for t, fmt, src in gallery_textures()]
    mats = mb.MaterialData(gallery_textured_materials(), tex, gpu_id=0)
    assert mats.view().num_texture_buffers == 3 and mats.view().texture_buffers
    rc = _RenderConfigC(0, bvh.view(device=True), mats.view(), 32, 0.001, 1000.0)
    desc = SIMS["gallery_textured"]
    saved = desc.render
    desc.render = lambda cfg: (rc, None)
    try:
        first = make_executor("gallery_textured", 2, num_props=30, seed=2)
        step, render = first.buildLaunchGraphAllTaskGraphs(), first.buildRenderGraph()
        first.run(step)
        first.run(render)
        del step, render
        first.close()
        a = make_executor("gallery_textured", 2, num_props=30, seed=2)
        b = make_executor("gallery_textured", 2, num_props=30, seed=2)
        images = []
        for ex in (a, b):
            step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
            ex.run(step)
            ex.run(render)
            images.append(ex.tensor(8, "uint8", (4, 32, 32, 4)).cpu().numpy())
            del step, render
        assert np.array_equal(images[0], images[1])
        a.close()
        b.close()
    finally:
        desc.render = saved
    mats.close()
    bvh.close()
    mats.close()          # closing twice is a no-op
