"""Float64 model of the narrowphase's contact classification (the reference's SAT path in
narrowphase.cpp, restated by kernels_physics.cu): for posed convex hulls it finds which
kind of contact a pair makes and how big the faces and clipped polygons involved are.
It does not reproduce the kernel's float32 results; it tells what a pose exercises, so a
fixture can be shown to reach the staging caps (tests/test_hull_contact_model.py)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np


def quat_matrix(q) -> np.ndarray:
    """Rotation matrix of a quaternion stored (w, x, y, z), as madrona's Quat."""
    w, x, y, z = (float(c) for c in q)
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


@dataclass
class Hull:
    verts: np.ndarray            # [V, 3] world space
    normals: np.ndarray          # [F, 3] unit, outward
    offsets: np.ndarray          # [F]
    faces: List[List[int]]       # vertex loops, counter-clockwise seen from outside
    edges: np.ndarray            # [E, 4]: vertex 0, vertex 1, face of half-edge 2k, face of its twin


def mesh_faces(mesh) -> List[List[int]]:
    he = mesh["half_edges"]
    loops = []
    for base in mesh["face_base"]:
        loop, h = [], int(base)
        while True:
            loop.append(int(he[h][1]))
            h = int(he[h][0])
            if h == int(base):
                break
        loops.append(loop)
    return loops


def pose_hull(mesh, pos, rot, scale) -> Hull:
    """vertex = R S v + t; face normal = normalize(R S^-1 n), offset through a posed point
    of the plane (narrowphase.cpp:151-223)."""
    r = quat_matrix(rot) if np.shape(rot) == (4,) else np.asarray(rot, dtype=np.float64)
    s = np.asarray(scale, dtype=np.float64)
    t = np.asarray(pos, dtype=np.float64)
    verts = (mesh["vertices"].astype(np.float64) * s) @ r.T + t
    local = mesh["planes"].astype(np.float64)
    normals = (local[:, :3] / s) @ r.T
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    on_plane = (local[:, :3] * local[:, 3:4] * s) @ r.T + t
    offsets = np.einsum("ij,ij->i", normals, on_plane)
    he = mesh["half_edges"]
    edges = np.array([[he[2 * k][1], he[he[2 * k][0]][1], he[2 * k][2], he[2 * k + 1][2]]
                      for k in range(len(he) // 2)], dtype=np.int64)
    return Hull(verts, normals, offsets, mesh_faces(mesh), edges)


def face_query(a: Hull, b: Hull):
    """(separation, face) of A's faces against B's vertices: the first face of largest
    separation."""
    seps = (b.verts @ a.normals.T).min(axis=0) - a.offsets
    f = int(np.argmax(seps))
    return float(seps[f]), f


def _arcs_cross(a, b, c, d):
    bxa, dxc = np.cross(b, a), np.cross(d, c)
    cba, dba = np.einsum("ij,ij->i", c, bxa), np.einsum("ij,ij->i", d, bxa)
    adc, bdc = np.einsum("ij,ij->i", a, dxc), np.einsum("ij,ij->i", b, dxc)
    return (cba * dba < 0) & (adc * bdc < 0) & (cba * bdc > 0)


def edge_query(a: Hull, b: Hull):
    """(separation, (edge of A, edge of B)) over the edge pairs whose Gauss-map arcs cross
    (the pairs forming a face of the Minkowski difference), normal pointing away from A's
    vertex centroid; (-inf, None) when no pair qualifies."""
    ea, eb = a.edges, b.edges
    ia, ib = np.meshgrid(np.arange(len(ea)), np.arange(len(eb)), indexing="ij")
    ia, ib = ia.ravel(), ib.ravel()
    cross = _arcs_cross(a.normals[ea[ia, 2]], a.normals[ea[ia, 3]],
                        -b.normals[eb[ib, 2]], -b.normals[eb[ib, 3]])
    ia, ib = ia[cross], ib[cross]
    if len(ia) == 0:
        return -np.inf, None
    pa, qa = a.verts[ea[ia, 0]], a.verts[ea[ia, 1]]
    pb, qb = b.verts[eb[ib, 0]], b.verts[eb[ib, 1]]
    axis = np.cross(qa - pa, qb - pb)
    length = np.linalg.norm(axis, axis=1)
    ok = length > 1e-12
    if not ok.any():
        return -np.inf, None
    axis, pa, pb, ia, ib = axis[ok] / length[ok, None], pa[ok], pb[ok], ia[ok], ib[ok]
    centre = a.verts.mean(axis=0)
    flip = np.einsum("ij,ij->i", axis, pa - centre) < 0
    axis[flip] *= -1
    seps = np.einsum("ij,ij->i", axis, pb - pa)
    k = int(np.argmax(seps))
    return float(seps[k]), (int(ia[k]), int(ib[k]))


def clip_polygon(points: np.ndarray, normal, offset) -> np.ndarray:
    """Sutherland-Hodgman against one plane, the side with n.p - d <= 0 kept."""
    out = []
    n = len(points)
    for i in range(n):
        v1, v2 = points[i - 1], points[i]
        d1, d2 = v1 @ normal - offset, v2 @ normal - offset
        if d1 <= 0 and d2 <= 0:
            out.append(v2)
        elif d1 <= 0 < d2 or d2 <= 0 < d1:
            out.append(v1 + (v2 - v1) * (-d1 / ((v2 - v1) @ normal)))
            if d2 <= 0:
                out.append(v2)
    return np.array(out).reshape(-1, 3)


@dataclass
class HullContact:
    kind: str                    # "face" or "edge"
    separation: float
    ref_is_a: bool = True
    ref_face: int = -1
    inc_face: int = -1
    ref_size: int = 0            # vertices of the reference face
    inc_size: int = 0            # vertices of the incident face
    clipped: int = 0             # points of the clipped incident polygon, before reduction


def hull_hull(a: Hull, b: Hull, margin: float = 0.0) -> Optional[HullContact]:
    """None when the pair is separated by more than `margin`; else the contact the SAT
    path makes: a face contact (reference face: the better face query, A's on a tie;
    incident face: the other hull's face most anti-parallel to it) unless an edge pair
    separates more than both face queries."""
    sep_a, face_a = face_query(a, b)
    if sep_a > margin:
        return None
    sep_b, face_b = face_query(b, a)
    if sep_b > margin:
        return None
    sep_e, _ = edge_query(a, b)
    if sep_e > margin:
        return None
    if sep_a <= sep_e and sep_b <= sep_e:
        return HullContact("edge", sep_e)
    ref_is_a = sep_a >= sep_b
    ref, inc, ref_face = (a, b, face_a) if ref_is_a else (b, a, face_b)
    inc_face = int(np.argmin(inc.normals @ ref.normals[ref_face]))
    loop = ref.faces[ref_face]
    poly = inc.verts[inc.faces[inc_face]]
    n_ref = ref.normals[ref_face]
    for i in range(len(loop)):
        cur, nxt = ref.verts[loop[i]], ref.verts[loop[(i + 1) % len(loop)]]
        side = np.cross(nxt - cur, n_ref)
        poly = clip_polygon(poly, side, side @ cur) if len(poly) else poly
    return HullContact("face", max(sep_a, sep_b), ref_is_a, ref_face, inc_face, len(loop),
                       len(inc.faces[inc_face]), len(poly))


@dataclass
class PlaneContact:
    inc_face: int
    inc_size: int                # vertices of the hull's face most anti-parallel to the plane
    below: int                   # of them, at or below the plane (+ margin)


def hull_plane(h: Hull, normal, offset, margin: float = 0.0) -> Optional[PlaneContact]:
    normal = np.asarray(normal, dtype=np.float64)
    if (h.verts @ normal).min() - offset > margin:
        return None
    f = int(np.argmin(h.normals @ normal))
    pts = h.verts[h.faces[f]]
    return PlaneContact(f, len(pts), int((pts @ normal - offset <= margin).sum()))


def sphere_hull(centre, radius: float, h: Hull, margin: float = 0.0) -> Optional[str]:
    """"inside" (the centre is inside the hull), "outside" (the sphere reaches the hull
    within margin) or None."""
    centre = np.asarray(centre, dtype=np.float64)
    dist = h.normals @ centre - h.offsets
    if dist.max() <= 0:
        return "inside"
    return "outside" if _point_hull_distance(centre, h) <= radius + margin else None


def _point_hull_distance(p, h: Hull) -> float:
    # nearest point on the hull's surface: over faces (inside the loop) and edges
    best = np.inf
    for f, loop in enumerate(h.faces):
        d = p @ h.normals[f] - h.offsets[f]
        q = p - d * h.normals[f]
        pts = h.verts[loop]
        inside = all(np.cross(pts[(i + 1) % len(pts)] - pts[i], q - pts[i]) @ h.normals[f] >= 0
                     for i in range(len(pts)))
        if inside:
            best = min(best, abs(d))
    for v0, v1, _, _ in h.edges:
        a, b = h.verts[v0], h.verts[v1]
        t = np.clip((p - a) @ (b - a) / ((b - a) @ (b - a)), 0.0, 1.0)
        best = min(best, float(np.linalg.norm(p - (a + t * (b - a)))))
    return best
