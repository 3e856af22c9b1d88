"""Panoramic views in the ray caster (mb2_render_config::projection = 1,
madrona_b200/csrc/kernels_render.cu).  CPU model of the kernel's float32 ray formula and of its
two culls for worlds of <= 64 instances, which replace the pinhole's frustum planes with cone
tests:

* the view cull drops a box whose bounding sphere lies wholly above or below the covered band
  of elevations, |phi| <= |atan(h)|;
* the tile cull keeps a box iff the angle between the tile's middle ray c and the box's centre
  is at most alpha + beta (alpha: half the tile's azimuth span plus half its elevation span over
  its pixel centres, widened by a quarter pixel; beta: the sphere's half-angle), compared in
  cosines, and always when alpha + beta >= pi.

Both must be CONSERVATIVE -- a box that any exact (float64) pixel ray enters may never be
dropped -- over random view rotations, fields of view (mirrored h < 0, near 0, up to 89 degrees
from the horizon) and boxes that contain the camera, straddle the seam behind it, sit at the
poles, just outside the elevation band, or are flat or degenerate.  The slacks are read from
the kernel source, so the model checks the constants the kernel is built with.  The ABI and the
C++ facade's overload are checked here too; tests/test_render_panorama.py runs the kernel."""
import os
import re
import subprocess

import numpy as np
import pytest

from test_raycast_aspect_culling_model import _random_rotation, pixel_rays, tile_shape

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PI = F(3.14159265358979)


def _kernel_constant(name):
    src = open(os.path.join(ROOT, "madrona_b200", "csrc", "kernels_render.cu")).read()
    m = re.search(r"constexpr float " + name + r" = ([0-9.eE+-]+)f;", src)
    assert m, name
    return F(float(m.group(1)))


BAND_SLACK = _kernel_constant("kPanoBandSlack")
CONE_SLACK = _kernel_constant("kPanoConeSlack")


def frame32(R):
    """the kernel's view frame in float32: u, forward from the rotation, vv = normalize(forward x u)"""
    uf, ff = R[:, 0].astype(F), R[:, 1].astype(F)
    vf = np.cross(ff, uf).astype(F)
    return uf, ff, (vf / np.sqrt(F((vf * vf).sum()))).astype(F)


def pano_rays32(uf, ff, vf, hf, W, H):
    """the kernel's panorama rays in float32, row-major [H * W, 3]"""
    phi_max = np.arctan(F(hf)).astype(F)
    s = F(-1) if hf < 0 else F(1)
    px = np.arange(W, dtype=F)
    py = np.arange(H, dtype=F)
    theta = (s * (F(2) * PI) * ((px + F(0.5)) / F(W) - F(0.5))).astype(F)
    phi = (F(2) * phi_max * ((py + F(0.5)) / F(H) - F(0.5))).astype(F)
    cp, sp = np.cos(phi)[:, None, None], np.sin(phi)[:, None, None]
    ct, st = np.cos(theta)[None, :, None], np.sin(theta)[None, :, None]
    d = (cp * (ct * ff + st * uf) + sp * vf).astype(F)
    d = (d / np.sqrt((d * d).sum(-1, keepdims=True))).astype(F)
    return d.reshape(-1, 3)


def pano_rays64(u, forward, vv, h, W, H):
    """the same rays in float64, row-major [H * W, 3]"""
    phi_max = np.arctan(h)
    s = -1.0 if h < 0 else 1.0
    theta = s * 2 * np.pi * ((np.arange(W) + 0.5) / W - 0.5)
    phi = 2 * phi_max * ((np.arange(H) + 0.5) / H - 0.5)
    cp, sp = np.cos(phi)[:, None, None], np.sin(phi)[:, None, None]
    d = cp * (np.cos(theta)[None, :, None] * forward + np.sin(theta)[None, :, None] * u) + sp * vv
    return (d / np.linalg.norm(d, axis=-1, keepdims=True)).reshape(-1, 3)


def pano_cones(lo, hi):
    """the kernel's panoCone for boxes [n, 3] (float32, relative to the view origin):
    (dir [n, 3], beta, sin beta, cos beta); beta = pi where the sphere holds the origin"""
    b = F(0.5) * (lo + hi)
    hh = F(0.5) * (hi - lo)
    r = np.sqrt((hh * hh).sum(1)).astype(F)
    d = np.sqrt((b * b).sum(1)).astype(F)
    inside = ~(d > r)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (F(1) / d).astype(F)
        direction = np.where(inside[:, None], F(0), b * inv[:, None]).astype(F)
        sinb = np.where(inside, F(0), np.minimum(r * inv, F(1))).astype(F)
    cosb = np.where(inside, F(-1), np.sqrt(np.maximum(F(1) - sinb * sinb, F(0)))).astype(F)
    beta = np.where(inside, PI, np.arcsin(sinb)).astype(F)
    return direction, beta, sinb, cosb


def view_keep(cones, vf, hf):
    """the kernel's panoOutsideBand, negated"""
    direction, beta = cones[0], cones[1]
    band = abs(np.arctan(F(hf)).astype(F))
    e = np.arcsin(np.clip((direction * vf).sum(1).astype(F), F(-1), F(1))).astype(F)
    outside = ((e - beta) > band + BAND_SLACK) | ((e + beta) < -band - BAND_SLACK)
    return (beta >= PI) | ~outside


def tile_cone(uf, ff, vf, hf, W, H, tx0, ty0):
    """the kernel's tile middle ray c and half-angle alpha (float32)"""
    tw, th = tile_shape(H)
    phi_max = np.arctan(F(hf)).astype(F)
    nx, ny = min(tw, W - tx0), min(th, H - ty0)
    s = F(-1) if hf < 0 else F(1)
    theta_c = F(s * (F(2) * PI) * ((F(tx0) + F(0.5) * F(nx)) / F(W) - F(0.5)))
    phi_c = F(F(2) * phi_max * ((F(ty0) + F(0.5) * F(ny)) / F(H) - F(0.5)))
    alpha = F((F(0.5) * F(nx - 1) + F(0.25)) * (F(2) * PI / F(W)) +
              (F(0.5) * F(ny - 1) + F(0.25)) * (F(2) * abs(phi_max) / F(H)))
    c = (np.cos(phi_c) * (np.cos(theta_c) * ff + np.sin(theta_c) * uf) + np.sin(phi_c) * vf).astype(F)
    return c, alpha


def tile_margin(cones, c, alpha):
    """dot(c, dir) - (cos alpha cos beta - sin alpha sin beta): the tile cull keeps a box where
    this is >= -CONE_SLACK; +inf where alpha + beta >= pi (always kept)"""
    direction, beta, sinb, cosb = cones
    dot = (direction * c).sum(1).astype(F)
    rhs = (np.cos(alpha) * cosb - np.sin(alpha) * sinb).astype(F)
    return np.where(alpha + beta >= PI, np.inf, dot - rhs)


# ---- the ray formula -------------------------------------------------------------------------------

def _angle(a, b):
    a = a.astype(np.float64)
    b = b.astype(np.float64)
    cr = np.linalg.norm(np.cross(a, b), axis=-1)
    return np.arctan2(cr, (a * b).sum(-1))


RAY_SIZES = [(1, 360), (16, 1024), (37, 5), (8, 3), (5, 7), (64, 64), (3, 9), (16, 256)]     # (H, W)


def test_float32_rays_match_float64_and_are_unit_length():
    rng = np.random.default_rng(3)
    for case in range(24):
        H, W = RAY_SIZES[case % len(RAY_SIZES)]
        R = _random_rotation(rng)
        h = [np.tan(np.radians(44.0)), -1.3, 1e-3, np.tan(np.radians(89.0)), -0.2, 0.0][case % 6]
        uf, ff, vf = frame32(R)
        d32 = pano_rays32(uf, ff, vf, F(h), W, H)
        # the float64 rays in the kernel's (float32) frame: the formula's own rounding only
        d64 = pano_rays64(uf.astype(np.float64), ff.astype(np.float64), vf.astype(np.float64), float(F(h)), W, H)
        assert _angle(d32, d64).max() < 1e-6, (H, W, h)
        assert np.abs(np.linalg.norm(d32.astype(np.float64), axis=1) - 1).max() < 1e-6


@pytest.mark.parametrize("h", [0.7, -0.7, 3.0, -0.05])
def test_centre_pixel_looks_forward_and_neighbours_turn_like_the_pinhole(h):
    rng = np.random.default_rng(11)
    R = _random_rotation(rng)
    u, forward = R[:, 0], R[:, 1]
    vv = np.cross(forward, u)
    uf, ff, vf = frame32(R)
    for H, W in [(5, 7), (37, 5), (3, 9), (1, 361), (9, 1)]:
        d = pano_rays32(uf, ff, vf, F(h), W, H).reshape(H, W, 3).astype(np.float64)
        pin = pixel_rays(u, forward, vv, h, W, H).reshape(H, W, 3)
        cy, cx = H // 2, W // 2
        assert _angle(d[cy, cx], forward) < 1e-6, (H, W)
        if W > 1:
            right = np.dot(d[cy, cx + 1] - d[cy, cx], u)
            assert np.sign(right) == np.sign(np.dot(pin[cy, cx + 1] - pin[cy, cx], u)) == np.sign(h)
        if H > 1:
            down = np.dot(d[cy + 1, cx] - d[cy, cx], vv)
            assert np.sign(down) == np.sign(np.dot(pin[cy + 1, cx] - pin[cy, cx], vv)) == np.sign(h)


def test_one_row_is_a_planar_scan_at_elevation_zero():
    rng = np.random.default_rng(4)
    for h in (0.0, 1e-4, 0.6, -2.0, np.tan(np.radians(89.0))):
        R = _random_rotation(rng)
        uf, ff, vf = frame32(R)
        for W in (360, 1024, 7):
            d = pano_rays32(uf, ff, vf, F(h), W, 1)
            assert np.abs(d.astype(np.float64) @ vf.astype(np.float64)).max() < 1e-7, (h, W)


def test_first_and_last_columns_mirror_about_the_backward_direction():
    rng = np.random.default_rng(8)
    for H, W in [(1, 360), (16, 1024), (5, 7), (37, 5), (8, 3)]:
        R = _random_rotation(rng)
        uf, ff, vf = frame32(R)
        for h in (0.9, -0.9):
            d = pano_rays32(uf, ff, vf, F(h), W, H).reshape(H, W, 3).astype(np.float64)
            a, b = d[:, 0], d[:, W - 1]
            f64, u64, v64 = ff.astype(np.float64), uf.astype(np.float64), vf.astype(np.float64)
            assert np.abs(a @ f64 - b @ f64).max() < 1e-6
            assert np.abs(a @ u64 + b @ u64).max() < 1e-6
            assert np.abs(a @ v64 - b @ v64).max() < 1e-6
            assert (a @ f64 < 0).all() and (b @ f64 < 0).all()        # both look backward


# ---- the culls are conservative ---------------------------------------------------------------------

def _boxes_entered(lo, hi, d):
    """exact slab test from the origin, t in [0, 1e4], boxes [n, 3] x rays [P, 3] -> bool [n, P]"""
    t0 = np.zeros((len(lo), len(d)))
    t1 = np.full((len(lo), len(d)), 1e4)
    ok = np.ones((len(lo), len(d)), dtype=bool)
    for a in range(3):
        da = d[None, :, a]
        zero = da == 0
        ok &= ~zero | ((lo[:, a, None] <= 0) & (0 <= hi[:, a, None]))
        with np.errstate(divide="ignore", invalid="ignore"):
            x, y = lo[:, a, None] / da, hi[:, a, None] / da
        t0 = np.where(zero, t0, np.maximum(t0, np.minimum(x, y)))
        t1 = np.where(zero, t1, np.minimum(t1, np.maximum(x, y)))
    return ok & (t0 <= t1)


CULL_SIZES = [(1, 360), (16, 1024), (37, 5), (5, 37), (8, 3), (5, 7), (64, 64)]      # (H, W)
H_VALUES = [-0.8, 1e-5, 0.0, 0.45, np.tan(np.radians(89.0)), -np.tan(np.radians(75.0)), 1.0, -3e-4]


def _boxes(rng, forward, u, vv, h):
    """boxes relative to the camera (float64 centres, half extents)"""
    c, half = [], []

    def add(centre, extent):
        c.append(np.asarray(centre, dtype=np.float64))
        half.append(np.asarray(extent, dtype=np.float64))
    for _ in range(20):                                      # all around
        add(rng.uniform(-12, 12, 3), rng.uniform(0.05, 4, 3))
    add(rng.uniform(-0.3, 0.3, 3), [0.5, 0.5, 0.5])          # contains the camera
    add([0.0, 0.0, 0.0], [0.0, 0.0, 0.0])                    # a point at the camera
    add(-8 * forward, [2.0, 2.0, 2.0])                       # straddles the seam behind it
    add(-30 * forward + 0.05 * u, [0.02, 0.02, 0.02])        # small, just beside the seam
    add(6 * vv, [0.3, 0.3, 0.3])                             # at the poles
    add(-6 * vv, [0.3, 0.3, 0.3])
    add(40 * vv + 0.01 * forward, [0.01, 0.01, 0.01])
    add([0.0, 0.0, 0.0], [1e4, 1e4, 0.5])                    # ground-plane slab
    add(rng.uniform(-8, 8, 3), [3.0, 2.0, 0.0])              # flat
    add(rng.uniform(-8, 8, 3), [0.0, 2.5, 0.0])              # a segment
    add(rng.uniform(-8, 8, 3), [0.0, 0.0, 0.0])              # a point
    band = abs(np.arctan(h))
    for sign in (1, -1):                                     # just outside / inside the band
        for delta in (2e-3, -2e-3, 5e-5):
            az = rng.uniform(-np.pi, np.pi)
            a, dist = rng.uniform(0.01, 0.5), rng.uniform(3, 20)
            beta = np.arcsin(min(1.0, a * np.sqrt(3) / dist))
            e = sign * (band + beta + delta)
            if abs(e) >= np.pi / 2:
                continue
            direction = np.cos(e) * (np.cos(az) * forward + np.sin(az) * u) + np.sin(e) * vv
            add(dist * direction, [a, a, a])
    return np.array(c), np.array(half)


def test_view_and_tile_culls_never_drop_a_box_a_pixel_ray_enters():
    rng = np.random.default_rng(29)
    needed_band, needed_cone = 0.0, 0.0
    entered_pairs, wide_pairs, culled_dense, pairs_dense = 0, 0, 0, 0
    for case in range(len(CULL_SIZES) * len(H_VALUES)):
        H, W = CULL_SIZES[case % len(CULL_SIZES)]
        h = H_VALUES[case // len(CULL_SIZES)]
        R = _random_rotation(rng)
        u, forward = R[:, 0], R[:, 1]
        vv = np.cross(forward, u)
        vv /= np.linalg.norm(vv)
        uf, ff, vf = frame32(R)
        hf = F(h)
        c, half = _boxes(rng, forward, u, vv, h)
        lo64, hi64 = c - half, c + half
        lo32, hi32 = lo64.astype(F), hi64.astype(F)
        cones = pano_cones(lo32, hi32)
        in_view = view_keep(cones, vf, hf)
        # the band test's margin without its slack, for the report below
        e = np.arcsin(np.clip((cones[0] * vf).sum(1), -1, 1))
        band = abs(np.arctan(hf))
        rays = pano_rays64(u, forward, vv, h, W, H).reshape(H, W, 3)
        # boxes shrunk by 1e-4 so that float32 rounding of a grazing ray does not count
        # (flat axes stay flat)
        shrink = np.minimum(1e-4 * (1 + np.abs(c)), half)
        tw, th = tile_shape(H)
        tiles_x = (W + tw - 1) // tw
        for tile in range(tiles_x * ((H + th - 1) // th)):
            tx0, ty0 = (tile % tiles_x) * tw, (tile // tiles_x) * th
            d = rays[ty0:ty0 + th, tx0:tx0 + tw].reshape(-1, 3)
            cc, alpha = tile_cone(uf, ff, vf, hf, W, H, tx0, ty0)
            margin = tile_margin(cones, cc, alpha)
            keep = in_view & (margin >= -CONE_SLACK)
            wide_pairs += int((np.isinf(margin) & (cones[1] < PI)).sum())
            entered = _boxes_entered(lo64 + shrink, hi64 - shrink, d).any(axis=1)
            for k in np.nonzero(entered)[0]:
                assert keep[k], (case, H, W, h, tile, k, bool(in_view[k]), float(margin[k]))
                entered_pairs += 1
                if cones[1][k] < PI:
                    needed_band = max(needed_band, e[k] - cones[1][k] - band, -band - e[k] - cones[1][k])
                needed_cone = max(needed_cone, -float(margin[k]))
            if (H, W) == (16, 1024):
                culled_dense += int((~keep).sum())
                pairs_dense += len(c)
    assert entered_pairs > 2000
    assert wide_pairs > 0          # tiles of small W reach alpha + beta >= pi with boxes outside
    # both slacks have room to spare: the GPU contracts to FMA where numpy rounds every step
    assert needed_band < 0.25 * BAND_SLACK, needed_band
    assert needed_cone < 0.25 * CONE_SLACK, needed_cone
    # the culls are not "keep all": most boxes leave most tiles of a 16 x 1024 panorama
    assert culled_dense > 0.6 * pairs_dense, (culled_dense, pairs_dense)


# ---- the C ABI and the C++ facade (no GPU needed) ----------------------------------------------------

def test_render_config_projection_matches_the_c_header(tmp_path):
    import ctypes
    from madrona_b200.executor import _RenderConfigC
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "madrona_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", sizeof(mb2_render_config), '
                   'offsetof(mb2_render_config, projection), offsetof(mb2_render_config, segmentation));'
                   ' return 0; }\n')
    exe = str(tmp_path / "layout")
    res = subprocess.run(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    size, proj_at, seg_at = (int(x) for x in subprocess.run([exe], capture_output=True, text=True,
                                                            check=True).stdout.split())
    assert ctypes.sizeof(_RenderConfigC) == size
    assert _RenderConfigC.projection.offset == proj_at
    assert proj_at == seg_at + 4                  # appended after segmentation


def test_invalid_projection_is_rejected_at_creation(monkeypatch):
    import madrona_b200 as mb
    from madrona_b200.executor import _MaterialViewC, _MeshBVHViewC, _RenderConfigC
    from sims import SIMS, make_executor
    rc = _RenderConfigC(0, _MeshBVHViewC(), _MaterialViewC(), 40, 0.001, 1000.0, 0, 0, 0, 2)
    monkeypatch.setattr(SIMS["gallery"], "render", lambda cfg: (rc, None))
    with pytest.raises(mb.MadronaB200Error, match=r"projection = 2 is not 0 \(pinhole\) or 1 \(panorama\)"):
        make_executor("gallery", 2, num_props=8)


def build_facade(tmp_path):
    exe = str(tmp_path / "facade_render_panorama")
    cmd = ["g++", "-std=c++20", "-O1", "-I" + os.path.join(ROOT, "madrona_b200", "host"),
           os.path.join(ROOT, "tests", "cpp", "facade_render_panorama.cpp"), "-o", exe,
           "-L" + os.path.join(ROOT, "madrona_b200"), "-lmadrona_b200",
           "-Wl,-rpath," + os.path.join(ROOT, "madrona_b200"),
           "-L/usr/local/cuda/lib64", "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    return exe


def test_facade_projection_overload_compiles(tmp_path):
    build_facade(tmp_path)
