"""What the large-hull narrowphase (MADRONA_B200_MAX_HULL_SIZE, physNarrowphaseLargeKernel)
rests on, shown on the CPU: the class of every fixture mesh as the device's primitive class
table must hold it; that the winner rule of the lane-strided scans gives the scalar scan's
answer for any lane count; that a polygon of n points clipped by m side planes holds at most
n + m points (the 2N-point clip buffers) unless rounding moves vertices across a side plane
they lie on; and that the hullpile_big goldens contain contacts of every pair kind the
feature adds (of sphere - large-hull pairs only the centre-outside kind).  CPU only."""
from collections import Counter

import numpy as np
import pytest

from hull_contact_model import hull_hull, hull_plane, pose_hull, sphere_hull
from sims.objects import box_half_edge_mesh, hull_size_class, hullpile_big_specs, hullpile_specs
from test_hull_clip_model import _ngon, _posed_pair, clip_face
from trace_utils import load_golden

# object index (SimObject order) -> class of its hull primitives at a knob of 16 / 32 / 64
SMALL3 = ("small", "small", "small")
PILE_CLASSES = {0: SMALL3, 1: SMALL3, 2: SMALL3, 3: SMALL3, 4: SMALL3, 5: SMALL3, 7: SMALL3, 8: SMALL3,
                10: SMALL3, 11: SMALL3}
BIG_CLASSES = dict(PILE_CLASSES)
BIG_CLASSES.update({
    2: ("too large", "too large", "large"),       # 24-gon prism: 48 vertices, 26 faces
    3: ("too large", "large", "large"),           # 16-gon bipyramid: 18 vertices, 32 faces
    4: ("too large", "too large", "too large"),   # icosphere: 42 vertices, 80 faces
    5: ("large", "large", "large"),               # 11-gon pyramid: 12 / 12, an 11-vertex base
    11: ("too large", "too large", "large"),
})


@pytest.mark.parametrize("specs,want", [(hullpile_specs, PILE_CLASSES), (hullpile_big_specs, BIG_CLASSES)],
                         ids=["hullpile", "hullpile_big"])
def test_primitive_classes(specs, want):
    for obj, sp in enumerate(specs()):
        for mesh in sp["prims"]:
            if isinstance(mesh, dict):
                got = tuple(hull_size_class(mesh, n) for n in (16, 32, 64))
                assert got == want[obj], (obj, got)
    assert hull_size_class(hullpile_big_specs()[4]["prims"][0], 80) == "large"


# ---- the winner rule -----------------------------------------------------------------------

def scalar_first_positive(values):
    """The reference's scan: keep strictly greater, stop at the first positive."""
    best, idx = -np.inf, None
    for i, v in enumerate(values):
        if v > best:
            best, idx = v, i
            if v > 0:
                break
    return idx


def strided_winner(values, lanes):
    """Each lane scans elements lane, lane + lanes, ... by the scalar rule; the reduction
    keeps the lowest index among positives, else the lowest index among maxima
    (groupSequentialWinner)."""
    picks = []
    for lane in range(lanes):
        mine = scalar_first_positive(values[lane::lanes])
        if mine is not None:
            picks.append(lane + mine * lanes)
    if not picks:
        return None
    positives = [i for i in picks if values[i] > 0]
    if positives:
        return min(positives)
    top = max(values[i] for i in picks)
    return min(i for i in picks if values[i] == top)


def test_winner_rule_does_not_depend_on_the_lane_count():
    rng = np.random.default_rng(5)
    cases = []
    for n in list(range(1, 40)) + [63, 64, 65, 127, 128, 200, 255]:
        cases.append(rng.normal(size=n).astype(np.float32))
        cases.append(-np.abs(rng.normal(size=n)).astype(np.float32))             # all negative
        cases.append(np.full(n, -0.25, dtype=np.float32))                        # all tied
        cases.append(np.round(rng.normal(size=n), 0).astype(np.float32) - 2)     # many ties
        one = -np.abs(rng.normal(size=n)).astype(np.float32)
        one[rng.integers(n)] = 0.5                                               # a single positive
        cases.append(one)
    for values in cases:
        want = scalar_first_positive(values)
        for lanes in (1, 4, 8, 32):
            assert strided_winner(values, lanes) == want, (len(values), lanes)


# ---- the clip bound ------------------------------------------------------------------------

def test_clip_stays_within_n_plus_m_points():
    # An n-gon clipped against the m side planes of an m-gon: a plane cuts a convex polygon
    # in at most two places, so every plane adds at most one point.  Generic poses (no
    # incident vertex on a side plane), around the yaw that cuts the most corners.
    worst = 0.0
    for n in range(3, 25):
        for m in range(3, 25):
            for yaw in (0.11, np.pi / m + 0.013, 0.37):
                inc, ref, up = _posed_pair(_ngon(n, yaw, radius=0.5), _ngon(m), np.eye(3))
                most = clip_face(inc, ref, up)[1]
                assert most <= n + m, (n, m, yaw, most)
                worst = max(worst, most / (n + m))
    assert worst == 1.0          # reached: a k-gon on a k-gon near pi / k makes 2k points


def test_rounding_can_exceed_n_plus_m_points():
    # A hexagon on a square with two shared corners: rounding puts vertices that lie on a side
    # plane on either side of it, a plane then cuts the polygon in more than two places, and
    # the count passes n + m.  This is why the kernel's clip keeps its "would not fit" check
    # even with 2N-point buffers for faces of at most N vertices.
    inc, ref, up = _posed_pair(_ngon(6, 0.0, radius=0.5), _ngon(4), np.eye(3))
    assert clip_face(inc, ref, up)[1] == 11


# ---- what the goldens exercise ----------------------------------------------------------------

STATIC = {9, 10, 11}
MARGIN = 0.01


def _pair_kinds(golden, stride):
    specs = hullpile_big_specs()
    large = {id(m): hull_size_class(m, 96) == "large"
             for sp in specs for m in sp["prims"] if isinstance(m, dict)}
    W, steps, _, outs = load_golden(golden)
    pos, rot = outs["body_pos"].astype(np.float64), outs["body_rot"].astype(np.float64)
    scale, obj = outs["body_scale"].astype(np.float64), outs["body_object"]
    counts = Counter()
    for t in range(0, steps + 1, stride):
        for w in range(W):
            prims = []       # (body, object, kind, posed, centre, reach, large)
            for b in range(pos.shape[2]):
                o = int(obj[t, w, b])
                for m in specs[o]["prims"]:
                    if isinstance(m, dict):
                        h = pose_hull(m, pos[t, w, b], rot[t, w, b], scale[t, w, b])
                        c = h.verts.mean(axis=0)
                        prims.append((b, o, "hull", h, c, np.linalg.norm(h.verts - c, axis=1).max(), large[id(m)]))
                    elif m == "plane":
                        n = pose_hull(box_half_edge_mesh(), (0, 0, 0), rot[t, w, b], (1, 1, 1)).normals[1]
                        prims.append((b, o, "plane", (n, float(n @ pos[t, w, b])), None, None, False))
                    else:
                        r = m[1] * scale[t, w, b, 0]
                        prims.append((b, o, "sphere", r, pos[t, w, b], r, False))
            for i in range(len(prims)):
                for j in range(i + 1, len(prims)):
                    pa, pb = prims[i], prims[j]
                    if pa[0] == pb[0] or (pa[1] in STATIC and pb[1] in STATIC):
                        continue
                    if pa[2] == "plane" or (pa[2] == "sphere" and pb[2] == "hull"):
                        pa, pb = pb, pa
                    if pa[2] != "hull":
                        continue
                    if pb[2] != "plane" and np.linalg.norm(pa[4] - pb[4]) > pa[5] + pb[5] + MARGIN:
                        continue
                    size = "large" if pa[6] else "small"
                    if pb[2] == "hull":
                        c = hull_hull(pa[3], pb[3], MARGIN)
                        if c is not None:
                            sizes = sorted([size, "large" if pb[6] else "small"])
                            counts[f"{sizes[0]}-{sizes[1]} {c.kind}"] += 1
                            if c.kind == "face" and c.clipped > 20:
                                counts["clipped past 20 points"] += 1
                            if c.kind == "face" and max(c.ref_size, c.inc_size) > 8:
                                counts["face over 8 vertices"] += 1
                    elif pb[2] == "plane":
                        c = hull_plane(pa[3], *pb[3], MARGIN)
                        if c is not None:
                            counts[f"{size}-plane"] += 1
                            if c.inc_size > 8:
                                counts["plane face over 8 vertices"] += 1
                    else:
                        c = sphere_hull(pb[4], pb[3], pa[3], MARGIN)
                        if c is not None:
                            counts[f"sphere-{size} {c}"] += 1
    return counts


def test_goldens_contain_every_large_pair_kind():
    pile = _pair_kinds("hullpile_big_w4_s150", 3)
    many = _pair_kinds("hullpile_big_many_w2_s100", 4)
    both = pile + many
    assert pile["large-large face"] >= 20 and both["large-large edge"] >= 5
    assert pile["large-small face"] >= 20 and both["large-small edge"] >= 5
    assert pile["small-small face"] + pile["small-small edge"] >= 20
    assert pile["large-plane"] >= 100 and pile["small-plane"] >= 100
    assert pile["plane face over 8 vertices"] >= 20
    assert pile["face over 8 vertices"] >= 20
    assert both["clipped past 20 points"] >= 1
    assert both["sphere-large inside"] + both["sphere-large outside"] >= 5
    assert both["sphere-small inside"] + both["sphere-small outside"] >= 5
