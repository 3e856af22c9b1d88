"""Ray caster culls for non-square images (madrona_b200/csrc/kernels_render.cu, worlds with <= 64
instances): the whole-view frustum, padded per axis, and the per-warp tile sub-frustum, for both
tile shapes (8 x 4, and 32 x 1 for images of fewer than 4 rows), must be CONSERVATIVE -- a box
that any pixel ray enters may never be dropped.  CPU model of the kernel's plane construction in
float32 against exact float64 rays over random cameras, fields of view (also mirrored, h < 0),
aspect ratios from 1/64 to 256, sizes that are not multiples of the tile, and boxes behind,
around and containing the camera.  For W == H the planes must be the square renderer's, bit for
bit (tests/test_raycast_culling_model.py restates those)."""
import numpy as np

F = np.float32


def _box_outside(lo, hi, n):
    c = F(0.5) * (lo + hi)
    h = F(0.5) * (hi - lo)
    reach = n[0] * c[0] + n[1] * c[1] + n[2] * c[2] + abs(n[0]) * h[0] + abs(n[1]) * h[1] + abs(n[2]) * h[2]
    return bool(reach < 0)


def _rays_enter(lo, hi, d):
    """exact slab test from the origin, t in [0, 1e4], rays d [P, 3] -> bool [P]"""
    t0, t1 = np.zeros(len(d)), np.full(len(d), 1e4)
    ok = np.ones(len(d), dtype=bool)
    for a in range(3):
        da = d[:, a]
        zero = da == 0
        ok &= ~zero | ((lo[a] <= 0) & (0 <= hi[a]))
        with np.errstate(divide="ignore", invalid="ignore"):
            x, y = lo[a] / da, hi[a] / da
        t0 = np.where(zero, t0, np.maximum(t0, np.minimum(x, y)))
        t1 = np.where(zero, t1, np.minimum(t1, np.maximum(x, y)))
    return ok & (t0 <= t1)


def _random_rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def tile_shape(H):
    """(tile width, tile height) of a warp: 32 x 1 below 4 rows, else 8 x 4"""
    return (32, 1) if H < 4 else (8, 4)


def view_planes(uf, ff, vf, hf, W, H):
    """the kernel's whole-view frustum normals (float32)"""
    aspect = F(W) / F(H)
    pad_u = abs(hf) * aspect * (F(1) + F(2) / F(W))
    pad_v = abs(hf) * (F(1) + F(2) / F(H))
    return [ff, uf + pad_u * ff, pad_u * ff - uf, vf + pad_v * ff, pad_v * ff - vf]


def tile_planes(uf, ff, vf, hf, W, H, tx0, ty0):
    """the kernel's tile sub-frustum normals (float32), edges a quarter pixel wider per axis"""
    tw, th = tile_shape(H)
    viewport = F(2) * hf
    viewport_w = viewport * (F(W) / F(H))
    inv_w, inv_h = F(1) / F(W), F(1) / F(H)
    a0 = (F(tx0) * inv_w - F(0.25) * inv_w - F(0.5)) * viewport_w
    a1 = (F(tx0 + tw) * inv_w + F(0.25) * inv_w - F(0.5)) * viewport_w
    b0 = (F(ty0) * inv_h - F(0.25) * inv_h - F(0.5)) * viewport
    b1 = (F(ty0 + th) * inv_h + F(0.25) * inv_h - F(0.5)) * viewport
    al, ar, bl, br = min(a0, a1), max(a0, a1), min(b0, b1), max(b0, b1)
    return [uf - al * ff, ar * ff - uf, vf - bl * ff, br * ff - vf]


def pixel_rays(u, forward, vv, h, W, H):
    """exact primary rays, row-major [H * W, 3]: vertical fov over the rows, horizontal half-extent
    h W / H"""
    pu = (np.arange(W) + 0.5) / W
    pv = (np.arange(H) + 0.5) / H
    d = (forward[None, None] + ((pu - 0.5) * 2 * h * W / H)[None, :, None] * u +
         ((pv - 0.5) * 2 * h)[:, None, None] * vv)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return d.reshape(-1, 3)


SIZES = [(64, 32), (32, 64), (40, 24), (37, 5), (256, 1), (1, 64), (8, 64), (45, 3), (130, 2), (13, 4),
         (24, 1), (3, 7)]


def test_aspect_view_and_tile_culls_never_drop_a_box_a_pixel_ray_enters():
    rng = np.random.default_rng(23)
    kept_and_hit, culled = 0, 0
    shapes_seen = set()
    for case in range(72):
        W, H = SIZES[case % len(SIZES)]
        R = _random_rotation(rng)
        u, forward = R[:, 0], R[:, 1]
        vv = np.cross(forward, u)
        vv /= np.linalg.norm(vv)
        h = np.tan(np.radians(rng.uniform(20, 120) * 0.5)) * (1 if case % 5 else -1)
        uf, ff, vf, hf = u.astype(F), forward.astype(F), vv.astype(F), F(h)
        # boxes relative to the camera: all around it, some containing it, some huge
        n = 24
        c = rng.uniform(-12, 12, size=(n, 3))
        half = rng.uniform(0.05, 4, size=(n, 3))
        half[0] = [1e4, 1e4, 0.5]                     # a ground-plane style slab
        c[1], half[1] = rng.uniform(-0.3, 0.3, 3), [0.5, 0.5, 0.5]     # contains the camera
        c[2] = -8 * forward                           # straight behind it
        lo64, hi64 = c - half, c + half
        lo32, hi32 = lo64.astype(F), hi64.astype(F)
        vplanes = view_planes(uf, ff, vf, hf, W, H)
        in_view = [not any(_box_outside(lo32[k], hi32[k], p) for p in vplanes) for k in range(n)]
        rays = pixel_rays(u, forward, vv, h, W, H).reshape(H, W, 3)
        # boxes shrunk by 1e-4 so that float32 rounding of a grazing ray does not count
        shrink = 1e-4 * (1 + np.abs(c))
        tw, th = tile_shape(H)
        shapes_seen.add((tw, th))
        tiles_x = (W + tw - 1) // tw
        for tile in range(tiles_x * ((H + th - 1) // th)):
            tx0, ty0 = (tile % tiles_x) * tw, (tile // tiles_x) * th
            planes = tile_planes(uf, ff, vf, hf, W, H, tx0, ty0)
            d = rays[ty0:ty0 + th, tx0:tx0 + tw].reshape(-1, 3)
            for k in range(n):
                keep = in_view[k] and not any(_box_outside(lo32[k], hi32[k], p) for p in planes)
                entered = _rays_enter(lo64[k] + shrink[k], hi64[k] - shrink[k], d)
                if entered.any():
                    assert keep, (case, W, H, tile, k)
                    kept_and_hit += int(entered.sum())
                culled += 0 if keep else 1
    assert shapes_seen == {(8, 4), (32, 1)}
    assert kept_and_hit > 20000 and culled > 5000     # both sides of the cull are exercised


def test_tile_grid_covers_every_pixel_once():
    for W, H in SIZES + [(4096, 1), (1, 1), (7, 3), (9, 4)]:
        tw, th = tile_shape(H)
        tiles_x = (W + tw - 1) // tw
        count = np.zeros((H, W), dtype=np.int64)
        for tile in range(tiles_x * ((H + th - 1) // th)):
            tx0, ty0 = (tile % tiles_x) * tw, (tile // tiles_x) * th
            shift = 5 if th == 1 else 3
            for lane in range(32):
                px, py = tx0 + (lane & (tw - 1)), ty0 + (lane >> shift)
                if px < W and py < H:
                    count[py, px] += 1
        assert (count == 1).all(), (W, H)


def _square_view_planes(uf, ff, vf, hf, res):
    """the square renderer's planes, as tests/test_raycast_culling_model.py states them"""
    pad = abs(hf) * (F(1) + F(2) / F(res))
    return [ff, uf + pad * ff, pad * ff - uf, vf + pad * ff, pad * ff - vf]


def _square_tile_planes(uf, ff, vf, hf, res, tx0, ty0):
    viewport = F(2) * hf
    inv_res = F(1) / F(res)
    a0 = (F(tx0) * inv_res - F(0.25) * inv_res - F(0.5)) * viewport
    a1 = (F(tx0 + 8) * inv_res + F(0.25) * inv_res - F(0.5)) * viewport
    b0 = (F(ty0) * inv_res - F(0.25) * inv_res - F(0.5)) * viewport
    b1 = (F(ty0 + 4) * inv_res + F(0.25) * inv_res - F(0.5)) * viewport
    al, ar, bl, br = min(a0, a1), max(a0, a1), min(b0, b1), max(b0, b1)
    return [uf - al * ff, ar * ff - uf, vf - bl * ff, br * ff - vf]


def test_square_planes_and_rays_are_bit_identical_to_the_square_renderer():
    rng = np.random.default_rng(5)
    for case in range(40):
        res = int(rng.choice([4, 16, 20, 37, 40, 64, 128, 1000]))
        R = _random_rotation(rng)
        uf, ff = R[:, 0].astype(F), R[:, 1].astype(F)
        vf = np.cross(ff, uf).astype(F)
        hf = F(np.tan(np.radians(rng.uniform(20, 120) * 0.5)) * (1 if case % 3 else -1))
        assert F(res) / F(res) == F(1)
        assert F(2) * hf * (F(res) / F(res)) == F(2) * hf
        for a, b in zip(view_planes(uf, ff, vf, hf, res, res), _square_view_planes(uf, ff, vf, hf, res)):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        assert tile_shape(res) == (8, 4)
        tiles_x = (res + 7) // 8
        for tile in range(0, tiles_x * ((res + 3) // 4), 7):
            tx0, ty0 = (tile % tiles_x) * 8, (tile // tiles_x) * 4
            for a, b in zip(tile_planes(uf, ff, vf, hf, res, res, tx0, ty0),
                            _square_tile_planes(uf, ff, vf, hf, res, tx0, ty0)):
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
