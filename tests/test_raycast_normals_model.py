"""Surface normals in the ray caster (mb2_render_config::normals = 1,
madrona_b200/csrc/kernels_render.cu encodeHitNormal).  CPU model of the kernel's float32 normal:
the hit triangle's object-space edge cross product, mapped to the world by M^T (M = the
instance's world -> object linear part, instanceXform), expressed in the view's frame
(x = n.u, y = n.vv, z = n.forward), turned against the ray, scaled to a largest component of 1,
normalised and encoded as round(127 n) clamped to +-127, w = 0.

It is checked against the float64 cross product of the triangle's world-space edges, within one
code per component, over non-uniform scales, mirrored instances (a negative scale component),
random view rotations, pinhole rays of mirrored views (h < 0), panorama rays and near-grazing
rays.  The C ABI layout, the rejection of normals = 2 and the C++ facade's RenderOutputs with
normals are checked here too; tests/test_render_normals.py runs the kernel."""
import os
import subprocess

import numpy as np
import pytest

from test_raycast_aspect_culling_model import _random_rotation, pixel_rays
from test_raycast_panorama_model import pano_rays64

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _quat(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def instance_xform32(q, scale):
    """instanceXform in float32: m = scale^-1 R(q)^T, row-major 3 x 3"""
    w, x, y, z = (F(c) for c in q)
    two = F(2)
    diag = F(1) - two * (x * x + y * y + z * z)
    R = np.array([[diag + two * x * x, two * (x * y - w * z), two * (x * z + w * y)],
                  [two * (x * y + w * z), diag + two * y * y, two * (y * z - w * x)],
                  [two * (x * z - w * y), two * (y * z + w * x), diag + two * z * z]], dtype=F)
    inv = (F(1) / scale.astype(F)).astype(F)
    return (R.T * inv[:, None]).astype(F)


def kernel_normal32(tri_obj, q, scale, u, vv, fwd, ray):
    """encodeHitNormal in float32: int8 [4] (x, y, z, w)"""
    a, b, c = (tri_obj[i].astype(F) for i in range(3))
    no = np.cross(b - a, c - a).astype(F)
    m = instance_xform32(q, scale)
    n = (m.T @ no).astype(F)
    s = F(-1) if F(n @ ray.astype(F)) > 0 else F(1)
    v = np.array([s * F(n @ u), s * F(n @ vv), s * F(n @ fwd)], dtype=F)
    big = F(np.abs(v).max())
    if not (big > 0 and np.isfinite(big)):
        return np.zeros(4, dtype=np.int8)
    v = (v * (F(1) / big)).astype(F)
    k = F(127) / F(np.sqrt(F((v * v).sum())))
    code = np.clip(np.rint((k * v).astype(F)), -127, 127).astype(np.int8)
    return np.concatenate([code, np.zeros(1, dtype=np.int8)])


def world_triangle64(tri_obj, q, scale, pos):
    """the instance's world-space triangle in float64 (tests/test_render_bvh.py's transform)"""
    w, x, y, z = q.astype(np.float64)
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                  [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    return tri_obj.astype(np.float64) @ (R * scale.astype(np.float64)[None, :]).T + pos


def oracle_normal64(tri_world, u, vv, fwd, ray):
    """(unit normal in the view frame turned against the ray, |cos| of the ray and the normal)"""
    n = np.cross(tri_world[1] - tri_world[0], tri_world[2] - tri_world[0])
    n /= np.linalg.norm(n)
    cos = float(n @ ray)
    if cos > 0:
        n = -n
    return np.array([n @ u, n @ vv, n @ fwd]), abs(cos)


def encode64(n):
    return np.clip(np.rint(127 * n), -127, 127).astype(np.int64)


def check(code, n64, cos):
    """one code per component of the float64 normal; where the ray grazes the surface
    (|cos| < 1e-4) either orientation"""
    assert code[3] == 0
    assert np.abs(code[:3].astype(np.int64)).max() >= 73           # never all zero on a hit
    got = code[:3].astype(np.int64)
    if np.abs(got - encode64(n64)).max() <= 1:
        return True
    assert cos < 1e-4 and np.abs(got - encode64(-n64)).max() <= 1, (got, encode64(n64), cos)
    return False


def _random_triangle(rng, size):
    return (rng.normal(size=(3, 3)) * size).astype(F)


def _random_scale(rng, mirrored):
    s = np.exp(rng.uniform(np.log(0.05), np.log(20.0), size=3))
    if mirrored:
        s[rng.integers(3)] *= -1
    return s.astype(F)


def _view(rng):
    """the kernel's view frame in float32 and float64: u, vv = normalize(forward x u), forward"""
    R = _random_rotation(rng)
    u, fwd = R[:, 0], R[:, 1]
    vv = np.cross(fwd, u)
    vv /= np.linalg.norm(vv)
    uf, ff = u.astype(F), fwd.astype(F)
    vf = np.cross(ff, uf).astype(F)
    vf = (vf / np.sqrt(F((vf * vf).sum()))).astype(F)
    return (uf, vf, ff), (u, vv, fwd)


# ---- the model against float64 world edges ------------------------------------------------------

@pytest.mark.parametrize("rays", ["pinhole", "pinhole_mirrored", "panorama", "panorama_mirrored"])
@pytest.mark.parametrize("mirrored", [False, True], ids=["scaled", "mirrored_instance"])
def test_float32_normal_matches_float64_world_edge_cross_product(rays, mirrored):
    rng = np.random.default_rng(11 + 2 * ["pinhole", "pinhole_mirrored", "panorama", "panorama_mirrored"].index(rays)
                                + int(mirrored))
    checked = 0
    for _ in range(60):
        (uf, vf, ff), (u, vv, fwd) = _view(rng)
        h = np.tan(np.radians(rng.uniform(10, 80) / 2)) * (-1 if rays.endswith("mirrored") else 1)
        W, H = int(rng.integers(1, 48)), int(rng.integers(1, 24))
        d64 = pano_rays64(u, fwd, vv, h, W, H) if rays.startswith("panorama") else pixel_rays(u, fwd, vv, h, W, H)
        for _ in range(8):
            q = _quat(rng)
            scale = _random_scale(rng, mirrored)
            tri = _random_triangle(rng, rng.uniform(0.01, 3.0))
            world = world_triangle64(tri, q, scale, rng.normal(size=3) * 5)
            ray = d64[rng.integers(len(d64))]
            n64, cos = oracle_normal64(world, u, vv, fwd, ray)
            code = kernel_normal32(tri, q, scale, uf, vf, ff, ray.astype(F))
            checked += check(code, n64, cos)
    assert checked > 0.99 * 60 * 8


def test_near_grazing_rays_keep_the_normal_and_orient_where_the_angle_is_resolved():
    """rays at 1e-7 .. 1e-2 rad from the triangle's plane: the normal's direction stays within
    one code, and its orientation is the float64 one wherever |cos| >= 1e-4"""
    rng = np.random.default_rng(5)
    oriented = 0
    for _ in range(400):
        (uf, vf, ff), (u, vv, fwd) = _view(rng)
        q = _quat(rng)
        scale = _random_scale(rng, bool(rng.integers(2)))
        tri = _random_triangle(rng, 1.0)
        world = world_triangle64(tri, q, scale, np.zeros(3))
        n = np.cross(world[1] - world[0], world[2] - world[0])
        n /= np.linalg.norm(n)
        t = world[1] - world[0]
        t /= np.linalg.norm(t)
        ang = 10.0 ** rng.uniform(-7, -2) * rng.choice([-1, 1])
        ray = np.cos(ang) * t + np.sin(ang) * n
        n64, cos = oracle_normal64(world, u, vv, fwd, ray)
        oriented += check(kernel_normal32(tri, q, scale, uf, vf, ff, ray.astype(F)), n64, cos)
    assert oriented > 100


def test_mirrored_instance_normal_is_the_world_edge_normal_not_the_rotated_object_normal():
    """a negative scale flips the triangle's winding in the world: M^T n_obj still points along
    the world edges' cross product (up to the sign the orientation removes), while the rotated
    object normal, which lighting uses, does not under non-uniform scale"""
    tri = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 1]], dtype=F)      # object normal -y
    q = np.array([1.0, 0.0, 0.0, 0.0])
    scale = np.array([-4.0, 1.0, 0.25], dtype=F)
    world = world_triangle64(tri, q, scale, np.zeros(3))
    u, vv, fwd = np.eye(3)[0], np.eye(3)[2], np.eye(3)[1]
    ray = np.array([0.0, 1.0, 0.0])
    n64, _ = oracle_normal64(world, u, vv, fwd, ray)
    code = kernel_normal32(tri, q, scale, u.astype(F), vv.astype(F), fwd.astype(F), ray.astype(F))
    assert np.array_equal(code, [0, 0, -127, 0])
    assert np.array_equal(encode64(n64), [0, 0, -127])

    # a sheared view of a tilted triangle: non-uniform scale moves the normal off the rotated one
    tri = np.array([[0, 0, 0], [1, 1, 0], [0, 0, 1]], dtype=F)
    scale = np.array([3.0, 1.0, 1.0], dtype=F)
    world = world_triangle64(tri, q, scale, np.zeros(3))
    n64, _ = oracle_normal64(world, u, vv, fwd, ray)
    code = kernel_normal32(tri, q, scale, u.astype(F), vv.astype(F), fwd.astype(F), ray.astype(F))
    assert np.abs(code[:3] - encode64(n64)).max() <= 1
    n_obj = np.cross(tri[1] - tri[0], tri[2] - tri[0]).astype(np.float64)
    n_obj /= np.linalg.norm(n_obj)
    if n_obj @ ray > 0:
        n_obj = -n_obj
    assert np.abs(encode64(n_obj) - encode64(n64)).max() > 10


def test_frame_and_orientation():
    """a wall square to the camera gives (0, 0, -127); tilting it toward +u (increasing
    column) and +vv (increasing row) makes x and y positive; either winding gives the same code"""
    u, vv, fwd = (v.astype(F) for v in np.eye(3))
    ray = fwd
    q = np.array([1.0, 0.0, 0.0, 0.0])
    one = np.ones(3, dtype=F)
    wall = np.array([[0, 0, 5], [1, 0, 5], [0, 1, 5]], dtype=F)       # the plane z = 5, forward = z
    assert np.array_equal(kernel_normal32(wall, q, one, u, vv, fwd, ray), [0, 0, -127, 0])
    assert np.array_equal(kernel_normal32(wall[::-1].copy(), q, one, u, vv, fwd, ray), [0, 0, -127, 0])
    # a surface whose outward normal leans toward +x and +y: (1, 1, -1) / sqrt 3
    tilted = np.array([[0, 0, 0], [1, 0, 1], [0, 1, 1]], dtype=F)
    code = kernel_normal32(tilted, q, one, u, vv, fwd, ray)
    assert np.array_equal(code, [73, 73, -73, 0])


def test_degenerate_triangle_encodes_to_zero():
    u, vv, fwd = (v.astype(F) for v in np.eye(3))
    q = np.array([1.0, 0.0, 0.0, 0.0])
    line = np.array([[0, 0, 0], [1, 1, 1], [2, 2, 2]], dtype=F)
    point = np.zeros((3, 3), dtype=F)
    for tri in (line, point):
        assert not kernel_normal32(tri, q, np.ones(3, dtype=F), u, vv, fwd, fwd).any()


def test_tiny_and_huge_triangles_keep_their_direction():
    """the scaling to a largest component of 1 before normalising keeps edges of 1e-12 (whose
    cross product squares underflow) and 1e12 (overflow) exact"""
    u, vv, fwd = (v.astype(F) for v in np.eye(3))
    q = np.array([1.0, 0.0, 0.0, 0.0])
    base = np.array([[0, 0, 0], [1, 0, 1], [0, 1, 1]], dtype=np.float64)
    for size in (1e-12, 1e-6, 1e6, 1e12):
        code = kernel_normal32((base * size).astype(F), q, np.ones(3, dtype=F), u, vv, fwd, fwd)
        assert np.array_equal(code, [73, 73, -73, 0]), size


# ---- the C ABI and the C++ facade (no GPU needed) ----------------------------------------------------

def test_render_config_normals_matches_the_c_header(tmp_path):
    import ctypes
    from madrona_b200.executor import _RenderConfigC
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "madrona_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu\\n", sizeof(mb2_render_config), '
                   'offsetof(mb2_render_config, normals), offsetof(mb2_render_config, projection));'
                   ' return 0; }\n')
    exe = str(tmp_path / "layout")
    res = subprocess.run(["gcc", "-std=c99", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    size, normals_at, proj_at = (int(x) for x in subprocess.run([exe], capture_output=True, text=True,
                                                                check=True).stdout.split())
    assert ctypes.sizeof(_RenderConfigC) == size
    assert _RenderConfigC.normals.offset == normals_at
    assert normals_at == proj_at + 4                # appended after projection


def test_invalid_normals_is_rejected_at_creation(monkeypatch):
    import madrona_b200 as mb
    from madrona_b200.executor import _MaterialViewC, _MeshBVHViewC, _RenderConfigC
    from sims import SIMS, make_executor
    rc = _RenderConfigC(0, _MeshBVHViewC(), _MaterialViewC(), 40, 0.001, 1000.0, 0, 0, 0, 0, 2)
    monkeypatch.setattr(SIMS["gallery"], "render", lambda cfg: (rc, None))
    with pytest.raises(mb.MadronaB200Error, match=r"normals = 2 is not 0 \(off\) or 1 \(on\)"):
        make_executor("gallery", 2, num_props=8)


def build_facade(tmp_path):
    exe = str(tmp_path / "facade_render_normals")
    cmd = ["g++", "-std=c++20", "-O1", "-I" + os.path.join(ROOT, "madrona_b200", "host"),
           os.path.join(ROOT, "tests", "cpp", "facade_render_normals.cpp"), "-o", exe,
           "-L" + os.path.join(ROOT, "madrona_b200"), "-lmadrona_b200",
           "-Wl,-rpath," + os.path.join(ROOT, "madrona_b200"),
           "-L/usr/local/cuda/lib64", "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    return exe


def test_facade_normals_output_compiles(tmp_path):
    build_facade(tmp_path)
