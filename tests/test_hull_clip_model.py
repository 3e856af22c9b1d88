"""Float32 model of the hull - hull face clip (kernels_physics.cu: clipAgainst and the
side-plane loop of hullHullGroup), one rounding per operation as the physics kernels
are built (--fmad=false, no contraction).

The clip buffers hold kClipCap = 2 * kMaxFaceVerts + 4 points.  Clipping a k-gon
against the k side planes of a k-gon can produce up to 2k points, so the buffers are
only safe because faces over kMaxFaceVerts vertices are refused before the clip.
These tests show both halves on the CPU: within the cap the largest intermediate
polygon fits over rotated, random and near-coincident aligned poses, and two 11-gon
faces (inside the 16-vertex / 16-face hull caps as the base of an 11-gon pyramid)
would not."""
import numpy as np
import pytest

f32 = np.float32
K_MAX_FACE_VERTS = 8
K_CLIP_CAP = 2 * K_MAX_FACE_VERTS + 4


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]          # left to right, as Vector3::dot


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _sub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def _lerp(v1, v2, d1, n):
    e = _sub(v2, v1)
    t = -d1 / _dot(n, e)
    return (v1[0] + e[0] * t, v1[1] + e[1] * t, v1[2] + e[2] * t)


def clip_against(src, normal, d):
    """Sutherland-Hodgman against one plane, "<= 0" inside (clipAgainst without its cap)."""
    out = []
    v1 = src[-1]
    d1 = _dot(v1, normal) - d
    for v2 in src:
        d2 = _dot(v2, normal) - d
        if d1 <= 0 and d2 <= 0:
            out.append(v2)
        elif d1 <= 0 and d2 > 0:
            out.append(_lerp(v1, v2, d1, normal))
        elif d2 <= 0 and d1 > 0:
            out.append(_lerp(v1, v2, d1, normal))
            out.append(v2)
        v1, d1 = v2, d2
    return out


def clip_face(incident, reference, ref_normal):
    """The incident polygon clipped against the side planes of the reference face (side
    normal = edge x n_ref, offset through the edge's first point), in the kernel's order.
    Returns (clipped polygon, largest point count any step held).  An incident edge
    that rounds to parallel with a side plane divides by zero, as in the kernel; the point
    count does not depend on the quotient."""
    src = list(incident)
    most = len(src)
    with np.errstate(all="ignore"):
        for i in range(len(reference)):
            cur, nxt = reference[i], reference[(i + 1) % len(reference)]
            side_n = _cross(_sub(nxt, cur), ref_normal)
            src = clip_against(src, side_n, _dot(side_n, cur)) if src else []
            most = max(most, len(src))
    return src, most


def _as32(p):
    return tuple(f32(c) for c in p)


def _rotate(rot, pts):
    return [_as32(rot @ np.asarray(p, dtype=np.float64)) for p in pts]


def _ngon(k, yaw=0.0, radius=0.5, z=0.0, scale=(1.0, 1.0), offset=(0.0, 0.0)):
    ang = yaw + 2.0 * np.pi * np.arange(k) / k
    return [(radius * scale[0] * np.cos(a) + offset[0], radius * scale[1] * np.sin(a) + offset[1], z)
            for a in ang]


def _random_rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _posed_pair(inc, ref, rot):
    """Reference face counter-clockwise about +z, incident face (on the other body, normal
    -z) clockwise, as the half-edge loops of two hulls meeting face to face; both posed by
    `rot` and rounded to float32 like the staged vertices."""
    up = _as32(rot @ np.array([0.0, 0.0, 1.0]))
    return _rotate(rot, inc[::-1]), _rotate(rot, ref), up


def test_model_clips_a_square_against_a_square_exactly():
    # a unit square over a larger one keeps its 4 corners; shifted half out, it is cut to 4
    ref = [_as32(p) for p in _ngon(4, np.pi / 4, radius=1.0)]
    up = _as32((0, 0, 1))
    inside = [_as32(p) for p in _ngon(4, np.pi / 4, radius=0.5)][::-1]
    pts, most = clip_face(inside, ref, up)
    assert len(pts) == 4 and most == 4
    assert sorted(pts) == sorted(inside)
    shifted = [_as32((x + 0.6, y, z)) for x, y, z in _ngon(4, np.pi / 4, radius=0.5)][::-1]
    pts, _ = clip_face(shifted, ref, up)
    xs = sorted(float(p[0]) for p in pts)
    assert len(pts) == 4 and xs[-1] == pytest.approx(np.sqrt(0.5), abs=1e-6)


@pytest.mark.parametrize("k", [3, 4, 5, 6, 7, 8])
def test_regular_faces_at_the_cap_rotated(k):
    # a k-gon on a k-gon at yaw pi/k cuts every corner: 2k points, 16 at the 8-vertex cap
    inc, ref, up = _posed_pair(_ngon(k, np.pi / k), _ngon(k), np.eye(3))
    pts, most = clip_face(inc, ref, up)
    assert len(pts) == 2 * k
    assert most <= K_CLIP_CAP
    rng = np.random.default_rng(k)
    for _ in range(60):
        inc, ref, up = _posed_pair(_ngon(k, rng.uniform(0, 2 * np.pi), radius=rng.uniform(0.3, 0.7)),
                                   _ngon(k, rng.uniform(0, 2 * np.pi)), _random_rotation(rng))
        assert clip_face(inc, ref, up)[1] <= K_CLIP_CAP


def test_random_faces_within_the_cap():
    # convex faces of 3..8 vertices (on ellipses, uneven angles), random sizes, offsets
    # and poses: no intermediate polygon exceeds the clip buffers
    rng = np.random.default_rng(7)
    worst = 0
    for _ in range(1500):
        polys = []
        for _side in range(2):
            k = int(rng.integers(3, K_MAX_FACE_VERTS + 1))
            ang = np.sort(rng.uniform(0, 2 * np.pi, size=k))
            sx, sy = rng.uniform(0.2, 1.0, size=2)
            ox, oy = rng.uniform(-0.3, 0.3, size=2)
            polys.append([(sx * np.cos(a) + ox, sy * np.sin(a) + oy, 0.0) for a in ang])
        inc, ref, up = _posed_pair(polys[0], polys[1], _random_rotation(rng))
        worst = max(worst, clip_face(inc, ref, up)[1])
    assert worst <= K_CLIP_CAP


@pytest.mark.parametrize("k", [4, 6, 8])
def test_near_coincident_aligned_faces_within_the_cap(k):
    # equal faces stacked with sub-micron misalignment (a box resting on a box, an 8-gon
    # on an 8-gon pedestal): every vertex sits on a side plane, so rounding decides
    # inside / outside; the count must still fit
    rng = np.random.default_rng(100 + k)
    worst = 0
    for t in range(1500):
        eps = rng.normal(size=2) * 10.0 ** rng.integers(-9, -5)
        yaw = rng.normal() * 10.0 ** rng.integers(-9, -5)
        rot = np.eye(3) if t % 2 == 0 else _random_rotation(rng)
        inc, ref, up = _posed_pair(_ngon(k, yaw, offset=eps), _ngon(k), rot)
        worst = max(worst, clip_face(inc, ref, up)[1])
    assert worst <= K_CLIP_CAP


@pytest.mark.parametrize("k,expect", [(11, 22), (15, 30)])
def test_faces_over_the_cap_overflow_the_clip_buffers(k, expect):
    # two 11-gon pyramid bases meeting at a relative yaw of pi/11: without the face-vertex
    # check the clip would write 22 points into 20-point buffers
    inc, ref, up = _posed_pair(_ngon(k, np.pi / k), _ngon(k), np.eye(3))
    pts, most = clip_face(inc, ref, up)
    assert len(pts) == expect and most == expect > K_CLIP_CAP
