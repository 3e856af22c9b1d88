"""Collision-object description for the rigid-body fixtures: builds the
madrona::phys::ObjectManager (include/madrona/physics.hpp:145-153 -- same
layout in this engine's device/madrona/physics.hpp) as ONE relocatable blob:
all arrays in a single buffer, pointer fields stored as offsets plus a
relocation list.  The oracle harness relocates it to host addresses, the GPU
path to device addresses, so both backends read identical geometry.

The reference builds this through PhysicsLoader + convex-hull processing
(src/physics/physics_assets.cpp, out of scope: SURVEY.md 8f N2); fixtures
hand-build boxes and a plane instead.
"""
from __future__ import annotations

import struct
from typing import List, Sequence, Tuple

import numpy as np

TYPE_SPHERE, TYPE_HULL, TYPE_PLANE = 1, 2, 4


def box_half_edge_mesh():
    """Unit cube [-0.5, 0.5]^3 as a half-edge mesh; twins are (2k, 2k+1)."""
    v = np.array([[x, y, z] for z in (-0.5, 0.5) for y in (-0.5, 0.5) for x in (-0.5, 0.5)],
                 dtype=np.float32)
    # CCW loops seen from outside
    faces = [
        [0, 2, 3, 1],   # -z
        [4, 5, 7, 6],   # +z
        [0, 1, 5, 4],   # -y
        [2, 6, 7, 3],   # +y
        [0, 4, 6, 2],   # -x
        [1, 3, 7, 5],   # +x
    ]
    return build_half_edge_mesh(v, faces)


def build_half_edge_mesh(verts: np.ndarray, faces: Sequence[Sequence[int]]):
    edge_ids = {}
    hedges: List[List[int]] = []          # [next, rootVertex, face], index = half-edge id
    face_base = []
    directed = {}
    for f, loop in enumerate(faces):
        n = len(loop)
        for i in range(n):
            a, b = loop[i], loop[(i + 1) % n]
            key = (min(a, b), max(a, b))
            if key not in edge_ids:
                edge_ids[key] = len(edge_ids)
                he = 2 * edge_ids[key]
            else:
                he = 2 * edge_ids[key] + 1
            assert (a, b) not in directed, "non-manifold"
            directed[(a, b)] = he
    n_he = 2 * len(edge_ids)
    hedges = [[0, 0, 0] for _ in range(n_he)]
    for f, loop in enumerate(faces):
        n = len(loop)
        ids = [directed[(loop[i], loop[(i + 1) % n])] for i in range(n)]
        face_base.append(ids[0])
        for i in range(n):
            hedges[ids[i]] = [ids[(i + 1) % n], loop[i], f]
    planes = []
    for loop in faces:
        p0, p1, p2 = verts[loop[0]], verts[loop[1]], verts[loop[2]]
        nrm = np.cross(p1 - p0, p2 - p0).astype(np.float64)
        nrm /= np.linalg.norm(nrm)
        nrm = nrm.astype(np.float32)
        planes.append([nrm[0], nrm[1], nrm[2], np.float32(np.dot(nrm, p0))])
    return dict(vertices=np.asarray(verts, dtype=np.float32),
                half_edges=np.asarray(hedges, dtype=np.uint32),
                face_base=np.asarray(face_base, dtype=np.uint32),
                planes=np.asarray(planes, dtype=np.float32))


class BlobBuilder:
    def __init__(self):
        self.buf = bytearray()
        self.relocs: List[int] = []

    def align(self, a: int):
        while len(self.buf) % a:
            self.buf.append(0)

    def add(self, data: bytes, align: int = 16) -> int:
        self.align(align)
        off = len(self.buf)
        self.buf += data
        return off

    def pointer_at(self, where: int, target_offset: int):
        struct.pack_into("<Q", self.buf, where, target_offset)
        self.relocs.append(where)


def _metadata(inv_mass, inv_inertia, mu_s, mu_d) -> bytes:
    # RigidBodyMassData {invMass, invInertiaTensor[3], toCenterOfMass[3], toInteriaFrame(w,x,y,z)}
    # + RigidBodyFrictionData {muS, muD}  = 52 bytes
    return struct.pack("<f3f3f4f2f", inv_mass, *inv_inertia, 0, 0, 0, 1, 0, 0, 0, mu_s, mu_d)


def room_objects(with_ball: bool = False) -> Tuple[bytes, List[int]]:
    """Objects of sims/room: 0 Cube, 1 Wall, 2 Agent, 3 Plane (one primitive each);
    with_ball appends 4 Ball (a sphere of radius 0.5) for sims/balls."""
    mesh = box_half_edge_mesh()
    b = BlobBuilder()
    mgr_off = b.add(b"\0" * 48)

    he_off = b.add(mesh["half_edges"].tobytes())
    fb_off = b.add(mesh["face_base"].tobytes())
    pl_off = b.add(mesh["planes"].tobytes())
    vt_off = b.add(mesh["vertices"].tobytes())

    n_obj = 5 if with_ball else 4
    prim_size = 56
    prims_off = b.add(b"\0" * (prim_size * n_obj), align=16)
    prim_types = [TYPE_HULL, TYPE_HULL, TYPE_HULL, TYPE_PLANE] + ([TYPE_SPHERE] if with_ball else [])
    for i, ty in enumerate(prim_types):
        base = prims_off + i * prim_size
        struct.pack_into("<I", b.buf, base, ty)
        if ty == TYPE_HULL:
            b.pointer_at(base + 8, he_off)
            b.pointer_at(base + 16, fb_off)
            b.pointer_at(base + 24, pl_off)
            b.pointer_at(base + 32, vt_off)
            struct.pack_into("<III", b.buf, base + 40, len(mesh["half_edges"]),
                             len(mesh["planes"]), len(mesh["vertices"]))
        elif ty == TYPE_SPHERE:
            struct.pack_into("<f", b.buf, base + 8, 0.5)      # CollisionPrimitive::sphere.radius

    hull_aabb = struct.pack("<6f", -0.5, -0.5, -0.5, 0.5, 0.5, 0.5)
    big = 1.0e5
    plane_aabb = struct.pack("<6f", -big, -big, -big, big, big, 0.0)
    aabbs = hull_aabb * 3 + plane_aabb + (hull_aabb if with_ball else b"")
    prim_aabb_off = b.add(aabbs)
    body_aabb_off = b.add(aabbs)
    offs_off = b.add(np.arange(n_obj, dtype=np.uint32).tobytes())
    cnts_off = b.add(np.ones(n_obj, dtype=np.uint32).tobytes())

    def box_inv_inertia(mass, sx, sy, sz):
        ix = mass / 12.0 * (sy * sy + sz * sz)
        iy = mass / 12.0 * (sx * sx + sz * sz)
        iz = mass / 12.0 * (sx * sx + sy * sy)
        return [np.float32(1.0 / ix), np.float32(1.0 / iy), np.float32(1.0 / iz)]

    cube_m, agent_m = 10.0, 50.0
    meta = b""
    meta += _metadata(np.float32(1.0 / cube_m), box_inv_inertia(cube_m, 1.5, 1.5, 1.5), 0.5, 0.75)
    meta += _metadata(0.0, [0.0, 0.0, 0.0], 0.5, 0.5)                      # wall (static)
    agent_inv_i = box_inv_inertia(agent_m, 1.0, 1.0, 1.5)
    meta += _metadata(np.float32(1.0 / agent_m), [0.0, 0.0, agent_inv_i[2]], 0.5, 0.5)  # yaw only
    meta += _metadata(0.0, [0.0, 0.0, 0.0], 0.5, 0.5)                      # plane
    if with_ball:
        # solid sphere used at scale 1.2 (radius 0.6): I = 2/5 m r^2
        ball_m, ball_r = 5.0, 0.6
        inv_i = np.float32(1.0 / (0.4 * ball_m * ball_r * ball_r))
        meta += _metadata(np.float32(1.0 / ball_m), [inv_i, inv_i, inv_i], 0.5, 0.5)
    meta_off = b.add(meta)

    for i, target in enumerate([prims_off, prim_aabb_off, body_aabb_off, offs_off, cnts_off, meta_off]):
        b.pointer_at(mgr_off + 8 * i, target)
    return bytes(b.buf), b.relocs


def balls_objects() -> Tuple[bytes, List[int]]:
    return room_objects(with_ball=True)


def relocate(blob: bytes, relocs: Sequence[int], base_address: int) -> bytes:
    out = bytearray(blob)
    for where in relocs:
        (off,) = struct.unpack_from("<Q", out, where)
        struct.pack_into("<Q", out, where, base_address + off)
    return bytes(out)


def write_blob_file(path: str, blob: bytes, relocs: Sequence[int]) -> None:
    """u64 size, u64 numRelocs, relocs[], blob (read by oracle/harness_room.cpp)."""
    with open(path, "wb") as f:
        f.write(struct.pack("<QQ", len(blob), len(relocs)))
        f.write(np.asarray(relocs, dtype=np.uint64).tobytes())
        f.write(blob)


# ---- generic builder (arbitrary convex hulls) ---------------------------------------------

def orient_faces(verts: np.ndarray, faces: Sequence[Sequence[int]]):
    """Reverse loops whose normal points at the hull centroid (=> CCW seen from outside)."""
    centroid = np.asarray(verts, dtype=np.float64).mean(axis=0)
    out = []
    for loop in faces:
        p = np.asarray([verts[i] for i in loop], dtype=np.float64)
        nrm = np.cross(p[1] - p[0], p[2] - p[0])
        out.append(list(loop) if np.dot(nrm, p.mean(axis=0) - centroid) > 0 else list(reversed(loop)))
    return out


def wedge_half_edge_mesh():
    """Unit ramp: right triangle in x-z (legs 1, right angle at the -x/-z corner)
    extruded along y; coordinates relative to the centroid."""
    t = 1.0 / 3.0
    tri = [(-t, -t), (2 * t, -t), (-t, 2 * t)]
    v = np.array([[x, y, z] for y in (-0.5, 0.5) for (x, z) in tri], dtype=np.float32)
    faces = [[0, 1, 2], [3, 4, 5], [0, 1, 4, 3], [0, 2, 5, 3], [1, 2, 5, 4]]
    return build_half_edge_mesh(v, orient_faces(v, faces))


def hex_prism_half_edge_mesh():
    """Unit hexagonal prism: circumradius 0.5, height 1 (12 vertices, 8 faces, 18 edges)."""
    s = 0.4330127
    ring = [(0.5, 0.0), (0.25, s), (-0.25, s), (-0.5, 0.0), (-0.25, -s), (0.25, -s)]
    v = np.array([[x, y, z] for z in (-0.5, 0.5) for (x, y) in ring], dtype=np.float32)
    faces = [list(range(6)), list(range(6, 12))] + [[i, (i + 1) % 6, (i + 1) % 6 + 6, i + 6] for i in range(6)]
    return build_half_edge_mesh(v, orient_faces(v, faces))


def bipyramid_half_edge_mesh(n: int = 8):
    """n-gon bipyramid: ring of circumradius 0.5 at z = 0, apexes at z = +-0.6 (n + 2
    vertices, 2n triangles, 3n edges; n = 8 is at the engine's 16-face hull cap)."""
    ang = 2.0 * np.pi * np.arange(n) / n
    v = np.array([[0.5 * np.cos(a), 0.5 * np.sin(a), 0.0] for a in ang] + [[0, 0, 0.6], [0, 0, -0.6]],
                 dtype=np.float32)
    faces = [[i, (i + 1) % n, n] for i in range(n)] + [[i, (i + 1) % n, n + 1] for i in range(n)]
    return build_half_edge_mesh(v, orient_faces(v, faces))


def pyramid_half_edge_mesh(n: int, apex=(0.0, 0.0)):
    """n-gon pyramid: base of circumradius 0.5 at z = -0.5, apex at (apex, 0.5) (n + 1
    vertices, n + 1 faces).  An off-centre apex leaves no two faces parallel."""
    ang = 2.0 * np.pi * np.arange(n) / n
    v = np.array([[0.5 * np.cos(a), 0.5 * np.sin(a), -0.5] for a in ang] + [[apex[0], apex[1], 0.5]],
                 dtype=np.float32)
    faces = [list(range(n))] + [[i, (i + 1) % n, n] for i in range(n)]
    return build_half_edge_mesh(v, orient_faces(v, faces))


def tetra_half_edge_mesh():
    """An irregular tetrahedron, vertices relative to their mean."""
    v = np.array([[0.55, -0.2, -0.3], [-0.4, 0.5, -0.3], [-0.3, -0.45, -0.25], [0.05, 0.1, 0.55]])
    v = (v - v.mean(axis=0)).astype(np.float32)
    return build_half_edge_mesh(v, orient_faces(v, [[0, 1, 2], [0, 1, 3], [1, 2, 3], [0, 2, 3]]))


def build_objects(specs, plane_extent: float = 1.0e5) -> Tuple[bytes, List[int]]:
    """specs: one dict per object -- {"mesh": <half-edge mesh dict> | "plane" | ("sphere", r),
    "meta": bytes(52)}; one primitive per object.  Same blob layout as room_objects()."""
    b = BlobBuilder()
    mgr_off = b.add(b"\0" * 48)
    mesh_offs = {}
    for sp in specs:
        m = sp["mesh"]
        if isinstance(m, dict) and id(m) not in mesh_offs:
            mesh_offs[id(m)] = (b.add(m["half_edges"].tobytes()), b.add(m["face_base"].tobytes()),
                                b.add(m["planes"].tobytes()), b.add(m["vertices"].tobytes()))
    n_obj = len(specs)
    prim_size = 56
    prims_off = b.add(b"\0" * (prim_size * n_obj), align=16)
    aabbs = b""
    big = plane_extent
    for i, sp in enumerate(specs):
        base = prims_off + i * prim_size
        m = sp["mesh"]
        if isinstance(m, dict):
            struct.pack_into("<I", b.buf, base, TYPE_HULL)
            he, fb, pl, vt = mesh_offs[id(m)]
            b.pointer_at(base + 8, he)
            b.pointer_at(base + 16, fb)
            b.pointer_at(base + 24, pl)
            b.pointer_at(base + 32, vt)
            struct.pack_into("<III", b.buf, base + 40, len(m["half_edges"]), len(m["planes"]),
                             len(m["vertices"]))
            lo, hi = m["vertices"].min(axis=0), m["vertices"].max(axis=0)
            aabbs += struct.pack("<6f", *lo, *hi)
        elif m == "plane":
            struct.pack_into("<I", b.buf, base, TYPE_PLANE)
            aabbs += struct.pack("<6f", -big, -big, -big, big, big, 0.0)
        else:
            struct.pack_into("<I", b.buf, base, TYPE_SPHERE)
            struct.pack_into("<f", b.buf, base + 8, float(m[1]))
            aabbs += struct.pack("<6f", *([-m[1]] * 3), *([m[1]] * 3))
    prim_aabb_off = b.add(aabbs)
    body_aabb_off = b.add(aabbs)
    offs_off = b.add(np.arange(n_obj, dtype=np.uint32).tobytes())
    cnts_off = b.add(np.ones(n_obj, dtype=np.uint32).tobytes())
    meta_off = b.add(b"".join(sp["meta"] for sp in specs))
    for i, target in enumerate([prims_off, prim_aabb_off, body_aabb_off, offs_off, cnts_off, meta_off]):
        b.pointer_at(mgr_off + 8 * i, target)
    return bytes(b.buf), b.relocs


def _box_inv_inertia(mass, sx, sy, sz):
    ix = mass / 12.0 * (sy * sy + sz * sz)
    iy = mass / 12.0 * (sx * sx + sz * sz)
    iz = mass / 12.0 * (sx * sx + sy * sy)
    return [np.float32(1.0 / ix), np.float32(1.0 / iy), np.float32(1.0 / iz)]


def arena_objects() -> Tuple[bytes, List[int]]:
    """Objects of sims/arena, in SimObject order: Cube, LongBox, Ramp, Barrel, Door, Wall,
    Pillar, Agent, Plane.  Inertia tensors are those of the bounding box at the scale the
    fixture uses the object at (the wedge / prism hulls are approximated by their boxes)."""
    box, wedge, hexp = box_half_edge_mesh(), wedge_half_edge_mesh(), hex_prism_half_edge_mesh()
    static = _metadata(0.0, [0.0, 0.0, 0.0], 0.5, 0.5)

    def dyn(mass, sx, sy, sz, mu_s=0.5, mu_d=0.5):
        return _metadata(np.float32(1.0 / mass), _box_inv_inertia(mass, sx, sy, sz), mu_s, mu_d)

    agent_m = 50.0
    agent_inv_i = _box_inv_inertia(agent_m, 1.0, 1.0, 1.5)
    specs = [
        dict(mesh=box, meta=dyn(10.0, 1.5, 1.5, 1.5, 0.5, 0.75)),            # Cube
        dict(mesh=box, meta=dyn(12.0, 2.4, 0.8, 1.0)),                       # LongBox
        dict(mesh=wedge, meta=dyn(15.0, 2.1, 2.0, 1.5)),                     # Ramp
        dict(mesh=hexp, meta=dyn(8.0, 1.2, 1.2, 1.2)),                       # Barrel
        dict(mesh=box, meta=dyn(20.0, 2.3, 0.3, 2.0)),                       # Door
        dict(mesh=box, meta=static),                                         # Wall
        dict(mesh=hexp, meta=static),                                        # Pillar
        dict(mesh=hexp, meta=_metadata(np.float32(1.0 / agent_m),            # Agent: yaw only
                                       [0.0, 0.0, agent_inv_i[2]], 0.5, 0.5)),
        dict(mesh="plane", meta=static),                                     # Plane
    ]
    return build_objects(specs)


def ngon_prism_half_edge_mesh(n: int):
    """Unit n-gon prism (2n vertices, n + 2 faces); n = 10 exceeds the engine's 16-vertex hull cap."""
    ang = 2.0 * np.pi * np.arange(n) / n
    ring = [(0.5 * np.cos(a), 0.5 * np.sin(a)) for a in ang]
    v = np.array([[x, y, z] for z in (-0.5, 0.5) for (x, y) in ring], dtype=np.float32)
    faces = [list(range(n)), list(range(n, 2 * n))] + [[i, (i + 1) % n, (i + 1) % n + n, i + n] for i in range(n)]
    return build_half_edge_mesh(v, orient_faces(v, faces))


def room_objects_big_hull() -> Tuple[bytes, List[int]]:
    """sims/room objects with the Cube replaced by a 20-vertex prism (tests/test_cliffs.py)."""
    box = box_half_edge_mesh()
    static = _metadata(0.0, [0.0, 0.0, 0.0], 0.5, 0.5)
    agent_inv_i = _box_inv_inertia(50.0, 1.0, 1.0, 1.5)
    specs = [
        dict(mesh=ngon_prism_half_edge_mesh(10),
             meta=_metadata(np.float32(0.1), _box_inv_inertia(10.0, 1.5, 1.5, 1.5), 0.5, 0.75)),
        dict(mesh=box, meta=static),
        dict(mesh=box, meta=_metadata(np.float32(1.0 / 50.0), [0.0, 0.0, agent_inv_i[2]], 0.5, 0.5)),
        dict(mesh="plane", meta=static),
    ]
    return build_objects(specs)


def build_compound_objects(specs, plane_extent: float = 1.0e5) -> Tuple[bytes, List[int]]:
    """specs: one dict per object -- {"prims": [<half-edge mesh dict> | "plane" | ("sphere", r),
    ...], "meta": bytes(52)}; an object may have several primitives (its body box is the union
    of theirs).  Same blob layout as build_objects()."""
    b = BlobBuilder()
    mgr_off = b.add(b"\0" * 48)
    prims = [p for sp in specs for p in sp["prims"]]
    mesh_offs = {}
    for m in prims:
        if isinstance(m, dict) and id(m) not in mesh_offs:
            mesh_offs[id(m)] = (b.add(m["half_edges"].tobytes()), b.add(m["face_base"].tobytes()),
                                b.add(m["planes"].tobytes()), b.add(m["vertices"].tobytes()))
    prim_size = 56
    prims_off = b.add(b"\0" * (prim_size * len(prims)), align=16)
    boxes = []
    big = plane_extent
    for i, m in enumerate(prims):
        base = prims_off + i * prim_size
        if isinstance(m, dict):
            struct.pack_into("<I", b.buf, base, TYPE_HULL)
            he, fb, pl, vt = mesh_offs[id(m)]
            b.pointer_at(base + 8, he)
            b.pointer_at(base + 16, fb)
            b.pointer_at(base + 24, pl)
            b.pointer_at(base + 32, vt)
            struct.pack_into("<III", b.buf, base + 40, len(m["half_edges"]), len(m["planes"]),
                             len(m["vertices"]))
            boxes.append((m["vertices"].min(axis=0), m["vertices"].max(axis=0)))
        elif m == "plane":
            struct.pack_into("<I", b.buf, base, TYPE_PLANE)
            boxes.append(([-big, -big, -big], [big, big, 0.0]))
        else:
            struct.pack_into("<I", b.buf, base, TYPE_SPHERE)
            struct.pack_into("<f", b.buf, base + 8, float(m[1]))
            boxes.append(([-m[1]] * 3, [m[1]] * 3))
    prim_aabb_off = b.add(b"".join(struct.pack("<6f", *lo, *hi) for lo, hi in boxes))
    body_boxes, offsets, counts, k = [], [], [], 0
    for sp in specs:
        n = len(sp["prims"])
        lo = np.min([boxes[k + j][0] for j in range(n)], axis=0)
        hi = np.max([boxes[k + j][1] for j in range(n)], axis=0)
        body_boxes.append(struct.pack("<6f", *lo, *hi))
        offsets.append(k)
        counts.append(n)
        k += n
    body_aabb_off = b.add(b"".join(body_boxes))
    offs_off = b.add(np.asarray(offsets, dtype=np.uint32).tobytes())
    cnts_off = b.add(np.asarray(counts, dtype=np.uint32).tobytes())
    meta_off = b.add(b"".join(sp["meta"] for sp in specs))
    for i, target in enumerate([prims_off, prim_aabb_off, body_aabb_off, offs_off, cnts_off, meta_off]):
        b.pointer_at(mgr_off + 8 * i, target)
    return bytes(b.buf), b.relocs


def shifted_box_half_edge_mesh(dx: float, dy: float, dz: float):
    """The unit cube of box_half_edge_mesh() moved by (dx, dy, dz) in object space."""
    box = box_half_edge_mesh()
    v = box["vertices"] + np.array([dx, dy, dz], dtype=np.float32)
    faces = [[0, 2, 3, 1], [4, 5, 7, 6], [0, 1, 5, 4], [2, 6, 7, 3], [0, 4, 6, 2], [1, 3, 7, 5]]
    return build_half_edge_mesh(v, faces)


def hullpile_objects(big_face: bool = False) -> Tuple[bytes, List[int]]:
    return build_compound_objects(hullpile_specs(big_face))


def hullpile_specs(big_face: bool = False):
    """Objects of sims/hullpile, in SimObject order: Box, Wedge, OctPrism (16 vertices, two
    8-vertex faces), Bipyramid (16 faces), Tetra, PentaPyramid (off-centre apex), Ball
    (radius 0.5), Dumbbell (two boxes 1.2 apart), CappedBox (a box below the origin and a
    sphere of radius 0.45 at it: a sphere primitive has no offset), Plane, Wall (static box),
    Pedestal (static octagonal prism).  Inertia tensors are those of the bounding box at unit
    scale.  big_face: OctPrism and Pedestal are 11-gon pyramids instead (12 vertices and 12
    faces, inside the hull caps, but an 11-vertex base: tests/test_cliffs.py)."""
    box, wedge = box_half_edge_mesh(), wedge_half_edge_mesh()
    prism = pyramid_half_edge_mesh(11) if big_face else ngon_prism_half_edge_mesh(8)
    static = _metadata(0.0, [0.0, 0.0, 0.0], 0.5, 0.5)

    def dyn(mass, sx, sy, sz):
        return _metadata(np.float32(1.0 / mass), _box_inv_inertia(mass, sx, sy, sz), 0.5, 0.5)

    ball_m, ball_r = 3.0, 0.5
    ball_inv_i = np.float32(1.0 / (0.4 * ball_m * ball_r * ball_r))
    specs = [
        dict(prims=[box], meta=dyn(4.0, 1.0, 1.0, 1.0)),                                     # Box
        dict(prims=[wedge], meta=dyn(4.0, 1.0, 1.0, 1.0)),                                   # Wedge
        dict(prims=[prism], meta=dyn(6.0, 1.0, 1.0, 1.0)),                                   # OctPrism
        dict(prims=[bipyramid_half_edge_mesh(8)], meta=dyn(4.0, 1.0, 1.0, 1.2)),            # Bipyramid
        dict(prims=[tetra_half_edge_mesh()], meta=dyn(2.0, 0.95, 0.95, 0.85)),               # Tetra
        dict(prims=[pyramid_half_edge_mesh(5, (0.15, 0.1))], meta=dyn(3.0, 1.0, 1.0, 1.0)),  # PentaPyramid
        dict(prims=[("sphere", ball_r)], meta=_metadata(np.float32(1.0 / ball_m),           # Ball
                                                        [ball_inv_i] * 3, 0.5, 0.5)),
        dict(prims=[shifted_box_half_edge_mesh(-0.6, 0.0, 0.0),                              # Dumbbell
                    shifted_box_half_edge_mesh(0.6, 0.0, 0.0)], meta=dyn(6.0, 2.2, 1.0, 1.0)),
        dict(prims=[shifted_box_half_edge_mesh(0.0, 0.0, -0.5), ("sphere", 0.45)],          # CappedBox
             meta=dyn(5.0, 1.0, 1.0, 1.45)),
        dict(prims=["plane"], meta=static),                                                  # Plane
        dict(prims=[box], meta=static),                                                      # Wall
        dict(prims=[prism], meta=static),                                                    # Pedestal
    ]
    return specs


def triggers_objects() -> Tuple[bytes, List[int]]:
    """Objects of sims/triggers, in SimObject order: Agent, Pickup, Wall, Floor (plane),
    Dumbbell (two unit boxes side by side along x, centred 0.6 from the origin: a compound
    of two hull primitives), Ball (a sphere of radius 0.5).  Bodies are kinematic or static:
    the fixture never runs the solver, so the mass data is nominal."""
    box = box_half_edge_mesh()
    static = _metadata(0.0, [0.0, 0.0, 0.0], 0.5, 0.5)
    specs = [
        dict(prims=[box], meta=static),                                            # Agent
        dict(prims=[box], meta=static),                                            # Pickup
        dict(prims=[box], meta=static),                                            # Wall
        dict(prims=["plane"], meta=static),                                        # Floor
        dict(prims=[shifted_box_half_edge_mesh(-0.6, 0.0, 0.0),
                    shifted_box_half_edge_mesh(0.6, 0.0, 0.0)], meta=static),      # Dumbbell
        dict(prims=[("sphere", 0.5)], meta=static),                                # Ball
    ]
    return build_compound_objects(specs)
