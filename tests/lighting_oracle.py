"""Float64 model of the batch ray caster's lighting (bvh_raycast.cpp:861-919, the light loop of
renderRaycastKernel in kernels_render.cu) for any list of lights.

Per hit and light: a directional light shines along -direction; a spotlight (LightDesc type
false) from its position, skipped outside its cone (acos of the angle to its direction above
|cutoff|) unless cutoff == -1 (a point light).  A light that casts shadows adds only if the
surface faces it and a shadow ray towards it, started 1 mm along the normal (the engine's one
deviation: the reference starts at the hit point itself), hits nothing in (1e-6, 10000) -- the
ray is not stopped at the light's position.  Each light adds clamp(n . l, 0, 1); the pixel is
min(1, max(0.2, sum) * base), truncated to 8 bits.  intensity and active are ignored, as the
reference ignores them.

`shade` also returns where float rounding may decide a pixel (the tolerances of the colour
checks in tests/test_render_bvh.py): a shadow ray whose result changes between origins 3e-4 and
3e-3 along the normal, a cone angle within 5e-3 of the cutoff, |n . l| < 5e-3 for a light that
casts shadows."""
from dataclasses import dataclass
from typing import List, Sequence

import numpy as np

from test_render_bvh import _closest_hits, _quat_rotate

SHADOW_OFFSET = 1e-3
SHADOW_T_MIN = 1e-6
SHADOW_T_MAX = 10000.0
GRAZE_OFFSETS = (3e-4, 3e-3)
EDGE_ANGLE = 5e-3
EDGE_NDOTL = 5e-3


@dataclass
class Light:
    """== render::LightDesc"""
    directional: bool
    cast_shadow: bool
    position: Sequence[float]
    direction: Sequence[float]
    cutoff: float
    intensity: float = 1.0
    active: bool = True


# the gallery fixture's two lamps (sims/gallery/sim.cpp)
GALLERY_LIGHTS = [
    Light(True, True, (0.0, 0.0, 9.0), (0.3, 0.2, -0.9327379), 0.9),
    Light(False, False, (0.0, 0.0, 9.0), (0.0, 0.0, -1.0), 0.9),
]


@dataclass
class Shading:
    value: np.ndarray       # [N, 3] float64 colour in [0, 1] before the 8-bit conversion
    rgb: np.ndarray         # [N, 3] uint8, truncated as the kernel converts
    edge: np.ndarray        # [N] bool: float rounding may decide the pixel
    beyond: np.ndarray      # [N] bool: a light's shadow ray is blocked only past the light
    shadowed: np.ndarray    # [N] bool: a facing light in range was blocked


def shadow_blocked(tris, origins, dirs):
    """any hit of the rays in (1e-6, 10000): [R] bool, and the closest t [R]"""
    if len(origins) == 0:
        return np.zeros(0, dtype=bool), np.zeros(0)
    t, _, _ = _closest_hits(origins, dirs, tris, t_min=SHADOW_T_MIN)
    return t < SHADOW_T_MAX, t


def shade(tris, hit_pos, normal, base, lights: List[Light]) -> Shading:
    """Colour of N hits: tris [T, 3, 3] the world's triangles (the shadow casters), hit_pos and
    normal [N, 3] (the engine's normal: the object-space geometric normal rotated by the
    instance rotation), base [N, 3] the surface colour, lights in any order."""
    hit_pos = np.asarray(hit_pos, dtype=np.float64).reshape(-1, 3)
    normal = np.asarray(normal, dtype=np.float64).reshape(-1, 3)
    base = np.asarray(base, dtype=np.float64).reshape(-1, 3)
    N = len(hit_pos)
    contrib = np.zeros(N)
    edge = np.zeros(N, dtype=bool)
    beyond = np.zeros(N, dtype=bool)
    shadowed = np.zeros(N, dtype=bool)
    for l in lights:
        d = np.asarray(l.direction, dtype=np.float64)
        inside = np.ones(N, dtype=bool)
        if l.directional:
            to_l = np.broadcast_to(-d, (N, 3)).copy()
            dist = np.full(N, np.inf)
        else:
            to_l = np.asarray(l.position, dtype=np.float64) - hit_pos
            dist = np.linalg.norm(to_l, axis=1)
            to_l /= dist[:, None]
            if l.cutoff != -1.0:
                cos_a = ((-to_l) @ d) / np.linalg.norm(d)
                ang = np.arccos(np.clip(cos_a, -1.0, 1.0))
                inside = np.abs(ang) <= abs(l.cutoff)
                edge |= np.abs(np.abs(ang) - abs(l.cutoff)) < EDGE_ANGLE
        ndl = (normal * to_l).sum(1)
        term = np.where(inside, np.clip(ndl, 0.0, 1.0), 0.0)
        if l.cast_shadow:
            edge |= inside & (np.abs(ndl) < EDGE_NDOTL)
            rows = np.nonzero(inside & (ndl > 0))[0]
            free = np.zeros(N, dtype=bool)
            if len(rows):
                o, dirs, nr = hit_pos[rows], to_l[rows], normal[rows]
                k = len(rows)
                # the three origins in one batch: the engine's, and the two graze probes
                origins = np.concatenate([o + SHADOW_OFFSET * nr] + [o + g * nr for g in GRAZE_OFFSETS])
                blocked, t = shadow_blocked(tris, origins, np.concatenate([dirs] * 3))
                b0, b1, b2 = blocked[:k], blocked[k:2 * k], blocked[2 * k:]
                free[rows] = ~b0
                edge[rows] |= (b0 != b1) | (b0 != b2)
                shadowed[rows] |= b0
                if not l.directional:
                    beyond[rows] |= b0 & (t[:k] > dist[rows])
            term = np.where(free, term, 0.0)
        contrib += term
    value = np.minimum(1.0, np.maximum(0.2, contrib)[:, None] * base)
    rgb = np.floor(value * 255.0).astype(np.uint8)
    return Shading(value, rgb, edge, beyond, shadowed)


def engine_normals(meshes, obj, rot, inst, src_tri):
    """the kernel's shading normal of hits on instance inst[i], triangle src_tri[i] of its mesh:
    the object-space unit normal rotated by the instance rotation (scale ignored, as the
    reference does)"""
    out = np.zeros((len(inst), 3))
    for j, (k, s) in enumerate(zip(inst, src_tri)):
        vtx, f, _ = meshes[int(obj[k])]
        a, b, c = vtx[f[s]].astype(np.float64)
        nn = np.cross(b - a, c - a)
        out[j] = _quat_rotate(rot[k].astype(np.float64), nn / np.linalg.norm(nn))
    return out


def base_colours(meshes, materials, obj, mat, color, inst):
    """the surface colour of hits on instance inst[i]: its colour override (material -2), else
    its material or its mesh's default material (-1); white for a mesh without one"""
    base = np.ones((len(inst), 3))
    for j, k in enumerate(inst):
        m = int(mat[k])
        if m == -2:
            hx = int(color[k])
            base[j] = [((hx >> 16) & 255) / 255.0, ((hx >> 8) & 255) / 255.0, (hx & 255) / 255.0]
            continue
        if m == -1:
            m = meshes[int(obj[k])][2]
        if m >= 0:
            base[j] = materials[m, :3]
    return base
