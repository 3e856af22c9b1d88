"""Render meshes of the rigid-body fixtures for the batch ray caster: one flat
triangle range per object ID (cube, wall, agent = unit box; plane = big quad).
The reference bakes MeshBVHs with embree (src/common/mesh_bvh_builder.cpp, not
available: SURVEY.md 8f N4); fixtures need a dozen triangles."""
from __future__ import annotations

import ctypes

import numpy as np


def unit_box():
    v = np.array([[x, y, z] for z in (-0.5, 0.5) for y in (-0.5, 0.5) for x in (-0.5, 0.5)],
                 dtype=np.float32)
    quads = [[0, 2, 3, 1], [4, 5, 7, 6], [0, 1, 5, 4], [2, 6, 7, 3], [0, 4, 6, 2], [1, 3, 7, 5]]
    tris = []
    for q in quads:
        tris += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
    return v, np.array(tris, dtype=np.uint32)


def room_meshes():
    """Returns (mesh_descs [n,8] float/uint view, vertices [nv,3] f32, indices [nt,3] u32)."""
    bv, bt = unit_box()
    e = 500.0
    pv = np.array([[-e, -e, 0], [e, -e, 0], [e, e, 0], [-e, e, 0]], dtype=np.float32)
    pt = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.uint32)
    verts = np.concatenate([bv, pv])
    plane_tris = pt + len(bv)
    indices = np.concatenate([bt, plane_tris])
    # objects: 0 cube, 1 wall, 2 agent share the box triangles; 3 = plane
    descs = np.zeros(4, dtype=[("first", "<u4"), ("count", "<u4"), ("mn", "<f4", 3), ("mx", "<f4", 3)])
    for o in range(3):
        descs[o] = (0, len(bt), (-0.5, -0.5, -0.5), (0.5, 0.5, 0.5))
    descs[3] = (len(bt), len(pt), (-e, -e, 0), (e, e, 0))
    return descs, verts, indices


def mesh_list(descs, verts, indices):
    """[(positions, triangles, material)] per object from the flat description."""
    out = []
    for d in descs:
        tris = indices[d["first"]:d["first"] + d["count"]]
        used = np.unique(tris)
        remap = {int(v): i for i, v in enumerate(used)}
        out.append((verts[used], np.vectorize(remap.get)(tris).astype(np.uint32), -1))
    return out


def make_render_config_from_meshes(meshes, resolution: int, rgbd: bool, gpu_id: int = 0, materials=None,
                                   width: int = 0, height: int = 0, segmentation: bool = False,
                                   panorama: bool = False, normals: bool = False):
    """mb2_render_config (== CudaBatchRenderConfig) whose geoBVHData was built by the
    engine's BLAS builder; returns (config, keep_alive).  width x height images when both are
    given (resolution then 0 or equal to both), else resolution squared.  segmentation: every
    view also gets an int32 image of hit entity ids.  panorama: every view is a 360-degree
    equirectangular panorama instead of a pinhole.  normals: every view also gets an int8 x 4
    image of the hit triangles' camera-facing normals in the view's frame."""
    import madrona_b200 as mb
    from madrona_b200.executor import _MaterialViewC, _RenderConfigC

    bvh = mb.MeshBVHData(meshes, gpu_id=gpu_id)
    mat_view = _MaterialViewC(None, 0, None, None)
    keep = [bvh]
    if materials is not None:
        import torch
        m = torch.from_numpy(np.ascontiguousarray(materials, dtype=np.float32)).to(f"cuda:{gpu_id}")
        keep.append(m)
        mat_view = _MaterialViewC(None, 0, None, m.data_ptr())
    rc = _RenderConfigC(0 if rgbd else 1, bvh.view(device=True), mat_view, resolution, 0.001, 1000.0,
                        width, height, int(segmentation), int(panorama), int(normals))
    return rc, keep


def make_render_config(resolution: int, rgbd: bool = False, gpu_id: int = 0, width: int = 0, height: int = 0,
                       segmentation: bool = False, panorama: bool = False, normals: bool = False):
    descs, verts, indices = room_meshes()
    return make_render_config_from_meshes(mesh_list(descs, verts, indices), resolution, rgbd, gpu_id,
                                          width=width, height=height, segmentation=segmentation,
                                          panorama=panorama, normals=normals)


# ---- gallery fixture: four prop meshes + ground ------------------------------------------------

def icosphere(subdiv: int = 2):
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
         [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11],
         [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    v = [np.array(p, dtype=np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(subdiv):
        cache, nf = {}, []

        def mid(a, b):
            key = (min(a, b), max(a, b))
            if key not in cache:
                m = (v[a] + v[b]) * 0.5
                v.append(m / np.linalg.norm(m))
                cache[key] = len(v) - 1
            return cache[key]
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return (np.array(v) * 0.5).astype(np.float32), np.array(f, dtype=np.uint32)


def prism(n: int):
    """n-gon prism with fans on the caps: 4n triangles."""
    ang = 2 * np.pi * np.arange(n) / n
    ring = np.stack([0.5 * np.cos(ang), 0.5 * np.sin(ang)], axis=1)
    v = [[x, y, -0.5] for x, y in ring] + [[x, y, 0.5] for x, y in ring] + [[0, 0, -0.5], [0, 0, 0.5]]
    f = []
    for i in range(n):
        j = (i + 1) % n
        f += [[i, j, j + n], [i, j + n, i + n], [2 * n, j, i], [2 * n + 1, i + n, j + n]]
    return np.array(v, dtype=np.float32), np.array(f, dtype=np.uint32)


def gallery_meshes():
    """[(positions, triangles, default material)]: box, icosphere (320 tris), 12-gon prism (48),
    tetrahedron (4), ground quad (2)."""
    bv, bt = unit_box()
    sv, st = icosphere(2)
    pv, pt = prism(12)
    tv = np.array([[0.5, 0.5, 0.5], [-0.5, -0.5, 0.5], [-0.5, 0.5, -0.5], [0.5, -0.5, -0.5]], dtype=np.float32)
    tt = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]], dtype=np.uint32)
    e = 60.0
    gv = np.array([[-e, -e, 0], [e, -e, 0], [e, e, 0], [-e, e, 0]], dtype=np.float32)
    gt = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.uint32)
    return [(bv, bt, 1), (sv, st, 2), (pv, pt, -1), (tv, tt, 3), (gv, gt, 0)]


GALLERY_MATERIALS = np.array([
    # color rgba, textureIdx (int bits), roughness, metalness  == madrona::Material (28 B)
    [0.55, 0.55, 0.5, 1.0, 0, 0.8, 0.0],
    [0.9, 0.3, 0.2, 1.0, 0, 0.5, 0.0],
    [0.2, 0.6, 0.9, 1.0, 0, 0.5, 0.0],
    [0.3, 0.8, 0.3, 1.0, 0, 0.5, 0.0],
], dtype=np.float32)
GALLERY_MATERIALS[:, 4] = np.array([-1], dtype=np.int32).view(np.float32)[0]     # textureIdx = -1


def make_gallery_render_config(resolution: int, rgbd: bool, gpu_id: int = 0, width: int = 0, height: int = 0,
                               segmentation: bool = False, panorama: bool = False, normals: bool = False):
    return make_render_config_from_meshes(gallery_meshes(), resolution, rgbd, gpu_id, materials=GALLERY_MATERIALS,
                                          width=width, height=height, segmentation=segmentation,
                                          panorama=panorama, normals=normals)


# ---- textured gallery: the same meshes with uvs, three generated textures -----------------------
# Pixels are made in code (decoding image files is the importer's job).  Each texture is built to
# catch one kind of mistake: the checker a wrong `1 - v` flip or barycentric order (8 x 8 with an
# asymmetric tint), the gradient swapped width and height (64 x 32), and the BC7 one the
# block-compressed upload path (mode-6 blocks, 16 x 16).

BC7_MODE6_WEIGHTS = np.array([0, 4, 9, 13, 17, 21, 26, 30, 34, 38, 43, 47, 51, 55, 60, 64], dtype=np.int64)


def _bc7_interp(e0, e1):
    """[..., 16 weights, 4] palette of a mode-6 block from 8-bit endpoints [..., 4]."""
    w = BC7_MODE6_WEIGHTS[:, None]
    return ((64 - w) * e0[..., None, :] + w * e1[..., None, :] + 32) >> 6


def bc7_mode6_encode(rgba):
    """RGBA8 [H, W, 4] (H, W multiples of 4) -> BC7 blocks uint8 [H/4, W/4, 16], mode 6 only:
    7-bit RGBA endpoints with one p-bit each, 4-bit indices.  The endpoints are the block's
    extremes along its principal axis, quantised with the p-bit pair of least error; every
    texel takes its nearest palette entry."""
    img = np.asarray(rgba, dtype=np.int64)
    H, W = img.shape[:2]
    assert img.shape[2] == 4 and H % 4 == 0 and W % 4 == 0
    out = np.zeros((H // 4, W // 4, 16), dtype=np.uint8)
    for by in range(H // 4):
        for bx in range(W // 4):
            px = img[by * 4:by * 4 + 4, bx * 4:bx * 4 + 4].reshape(16, 4)
            mean = px.mean(0)
            axis = np.linalg.eigh(np.cov((px - mean).T) + 1e-9 * np.eye(4))[1][:, -1]
            proj = (px - mean) @ axis
            ends = np.clip([mean + proj.min() * axis, mean + proj.max() * axis], 0, 255)
            best = None
            for p0 in (0, 1):
                for p1 in (0, 1):
                    c0 = np.clip(np.round((ends[0] - p0) / 2), 0, 127).astype(np.int64)
                    c1 = np.clip(np.round((ends[1] - p1) / 2), 0, 127).astype(np.int64)
                    pal = _bc7_interp((c0 << 1) | p0, (c1 << 1) | p1)
                    d = ((px[:, None, :] - pal[None]) ** 2).sum(-1)
                    err = d.min(1).sum()
                    if best is None or err < best[0]:
                        best = (err, c0, c1, p0, p1, d.argmin(1))
            _, c0, c1, p0, p1, idx = best
            if idx[0] >= 8:           # the anchor index has 3 bits: swap the endpoints
                c0, c1, p0, p1 = c1, c0, p1, p0
                idx = 15 - idx
            bits = 1 << 6             # mode 6
            pos = 7
            for ch in range(4):
                for c in (c0, c1):
                    bits |= int(c[ch]) << pos
                    pos += 7
            bits |= p0 << pos
            bits |= p1 << (pos + 1)
            pos += 2
            for i in range(16):
                bits |= int(idx[i]) << pos
                pos += 3 if i == 0 else 4
            assert pos == 128
            out[by, bx] = np.frombuffer(bits.to_bytes(16, "little"), dtype=np.uint8)
    return out


def bc7_mode6_decode(blocks):
    """BC7 mode-6 blocks uint8 [H/4, W/4, 16] -> RGBA8 [H, W, 4] (the format's exact decode)."""
    blocks = np.asarray(blocks, dtype=np.uint8)
    bh, bw = blocks.shape[:2]
    out = np.zeros((bh * 4, bw * 4, 4), dtype=np.uint8)
    for by in range(bh):
        for bx in range(bw):
            bits = int.from_bytes(blocks[by, bx].tobytes(), "little")
            assert bits & 0x7F == 1 << 6, "not a mode-6 block"
            pos = 7
            c = np.zeros((2, 4), dtype=np.int64)
            for ch in range(4):
                for e in range(2):
                    c[e, ch] = (bits >> pos) & 0x7F
                    pos += 7
            p = [(bits >> pos) & 1, (bits >> (pos + 1)) & 1]
            pos += 2
            pal = _bc7_interp((c[0] << 1) | p[0], (c[1] << 1) | p[1])
            for i in range(16):
                n = 3 if i == 0 else 4
                out[by * 4 + i // 4, bx * 4 + i % 4] = pal[(bits >> pos) & ((1 << n) - 1)]
                pos += n
    return out


def checker_texture():
    """8 x 8 RGBA8 checker: dark cells, light cells tinted by column and row."""
    i, j = np.meshgrid(np.arange(8), np.arange(8))          # i: column (u), j: row
    light = np.stack([np.full((8, 8), 255), 255 - 24 * i, 255 - 24 * j, np.full((8, 8), 255)], -1)
    dark = np.broadcast_to(np.array([16, 16, 40, 255]), (8, 8, 4))
    return np.where(((i + j) % 2 == 0)[..., None], light, dark).astype(np.uint8)


def gradient_texture():
    """64 wide x 32 high smooth RGBA8 gradient."""
    x, y = np.meshgrid(np.arange(64), np.arange(32))
    return np.stack([np.round(255 * x / 63), np.round(255 * y / 31), np.round(60 + 3 * (x + y) / 2),
                     np.full(x.shape, 255)], -1).astype(np.uint8)


def bc7_source_image():
    """16 x 16 RGBA8 image the BC7 texture is encoded from."""
    x, y = np.meshgrid(np.arange(16), np.arange(16))
    return np.stack([16 * x + 8, 255 - 12 * y, 128 + 7 * (x - y), np.full(x.shape, 255)], -1).astype(np.uint8)


def gallery_textures():
    """[(texels RGBA8 [H, W, 4] as sampled, format, source bytes)]: checker, gradient, BC7."""
    bc7 = bc7_mode6_encode(bc7_source_image())
    return [(checker_texture(), 0, checker_texture().tobytes()),
            (gradient_texture(), 0, gradient_texture().tobytes()),
            (bc7_mode6_decode(bc7), 1, bc7.tobytes())]


def _planar_uvs(v, scale):
    """uv linear in the position (no box face maps to a line), centred on 0.5."""
    v = np.asarray(v, dtype=np.float64)
    return np.stack([scale * (v[:, 0] + 0.5 * v[:, 2]) + 0.5, scale * (v[:, 1] - 0.5 * v[:, 2]) + 0.5],
                    1).astype(np.float32)


def gallery_textured_meshes():
    """gallery_meshes() with uvs: props mapped planar (uvs about [-1, 2], so they wrap), the
    ground quad's corners at uv 0 and 6."""
    out = []
    for k, (v, f, mat) in enumerate(gallery_meshes()):
        if k == 4:
            uv = np.array([[0, 0], [6, 0], [6, 6], [0, 6]], dtype=np.float32)
        else:
            uv = _planar_uvs(v, 1.5)
        out.append((v, f, mat, uv))
    return out


def gallery_textured_materials(bc7: bool = False):
    """GALLERY_MATERIALS' colours; material 0 (the ground's override) samples the checker,
    material 2 (the icosphere's default) the gradient, or with bc7 the BC7 texture."""
    tex_of = {0: 0, 2: 2 if bc7 else 1}
    return [(tuple(float(c) for c in m[:4]), tex_of.get(i, -1), float(m[5]), float(m[6]))
            for i, m in enumerate(GALLERY_MATERIALS)]


def make_gallery_textured_render_config(resolution: int, rgbd: bool, gpu_id: int = 0, bc7: bool = False,
                                        width: int = 0, height: int = 0, segmentation: bool = False,
                                        panorama: bool = False, normals: bool = False):
    """CudaBatchRenderConfig with textured materials uploaded by mb2_init_material_data; the
    MaterialData in keep_alive must outlive the executor."""
    import madrona_b200 as mb
    from madrona_b200.executor import _RenderConfigC

    bvh = mb.MeshBVHData(gallery_textured_meshes(), gpu_id=gpu_id)
    textures = [(src, fmt, t.shape[1], t.shape[0]) for t, fmt, src in gallery_textures()]
    mats = mb.MaterialData(gallery_textured_materials(bc7), textures, gpu_id=gpu_id)
    rc = _RenderConfigC(0 if rgbd else 1, bvh.view(device=True), mats.view(), resolution, 0.001, 1000.0,
                        width, height, int(segmentation), int(panorama), int(normals))
    return rc, [bvh, mats]
