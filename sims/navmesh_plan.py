"""Floor plans of the navmesh fixture, as sims/navmesh/plan.hpp builds them (the two must
stay in step: tests/test_navmesh.py checks this port against the C++ generator)."""
from __future__ import annotations

import numpy as np

GRID = 6
WALL_COLUMN = 4
SHARED_PLAN_SEED = 0x5EED
M32 = 0xFFFFFFFF


def plan_hash(seed: int, i: int) -> int:
    x = (seed * 0x9E3779B9 + i * 0x85EBCA6B + 0x165667B1) & M32
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & M32
    x ^= x >> 16
    return x


def make_plan(seed: int, bad_polygon: bool = False):
    """(vertices [nv,3] float32, polygons: list of index loops)"""
    verts = []
    polys = []

    def vert(x, y, z):
        verts.append((x, y, z))
        return len(verts) - 1

    def lat(i, j):
        return j * (GRID + 1) + i

    for j in range(GRID + 1):
        for i in range(GRID + 1):
            vert(float(i), float(j), 0.0)
    apex = vert(2.5, 2.0, 1.0)
    polys.append([lat(0, 0), lat(1, 0), lat(2, 0), lat(2, 1), lat(1, 1), lat(0, 1)])

    door = plan_hash(seed, 1000) % (GRID + 2)
    pentagons = 0
    for j in range(GRID):
        for i in range(GRID):
            if j == 0 and i < 2:
                continue
            a, b, c, d = lat(i, j), lat(i + 1, j), lat(i + 1, j + 1), lat(i, j + 1)
            fixed = i == 2 and j in (1, 2)
            if not fixed:
                if i == WALL_COLUMN and j != door:
                    continue
                r = plan_hash(seed, j * GRID + i) % 8
                if r == 0:
                    continue
                if r == 1:
                    m = vert(float(i + 1), float(j) + 0.5, 0.0)
                    polys.append([a, b, m, c, d])
                    pentagons += 1
                    continue
            polys.append([a, b, c, d])

    polys.append([lat(2, 2), lat(3, 2), apex])
    for k in range(pentagons):
        x, y = float(GRID + 1), float(2 * k)
        polys.append([vert(x, y, 0.0), vert(x + 2.0, y, 0.0), vert(x, y + 1.0, 0.0)])
    if bad_polygon:
        polys.append([lat(0, 0), lat(1, 0)])
    return np.asarray(verts, dtype=np.float32), polys
