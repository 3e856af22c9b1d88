"""The float64 contact model (tests/hull_contact_model.py) on poses whose answer is known,
then over every frame of the sims/hullpile goldens: the fixture must reach what the
narrowphase's lane-strided scans and staging caps are sized for -- 8-vertex reference
faces clipped to more than 8 points, every face of a 16-face hull, edge - edge pairs,
8-point hull - plane incident faces, spheres with their centre inside and outside hulls,
both primitives of both compound bodies, and (60-body variant) hull contacts on bodies
past the 48 the position solve stages in shared memory.  CPU only."""
from collections import Counter

import numpy as np
import pytest

from hull_contact_model import hull_hull, hull_plane, pose_hull, sphere_hull
from sims.objects import (bipyramid_half_edge_mesh, box_half_edge_mesh, hullpile_specs,
                          ngon_prism_half_edge_mesh, tetra_half_edge_mesh)
from trace_utils import load_golden

IDENTITY = (1.0, 0.0, 0.0, 0.0)
UP = np.array([0.0, 0.0, 1.0])


def _yaw(angle):
    return (np.cos(angle / 2), 0.0, 0.0, np.sin(angle / 2))


def test_box_resting_on_a_box():
    box = box_half_edge_mesh()
    below = pose_hull(box, (0, 0, 0.5), IDENTITY, (2, 2, 1))
    above = pose_hull(box, (0.1, 0.2, 1.495), _yaw(0.3), (1, 1, 1))
    c = hull_hull(above, below)
    assert c.kind == "face" and c.separation == pytest.approx(-0.005)
    # both face queries find 5 mm: A's bottom face is the reference on the tie, B's top face
    # is clipped to it
    assert c.ref_is_a and c.ref_size == 4 and c.inc_size == 4 and c.clipped == 4
    assert c.ref_face == 0 and c.inc_face == 1
    assert hull_hull(pose_hull(box, (0, 0, 1.6), IDENTITY, (1, 1, 1)), below) is None
    assert hull_hull(pose_hull(box, (0, 0, 1.6), IDENTITY, (1, 1, 1)), below, margin=0.11) is not None


def test_crossed_edges():
    # two unit cubes turned 45 degrees about x and about y: their ridges cross at 90 degrees
    box = box_half_edge_mesh()
    c, s = np.cos(np.pi / 8), np.sin(np.pi / 8)
    a = pose_hull(box, (0, 0, 0), (c, s, 0, 0), (1, 1, 1))
    b = pose_hull(box, (0, 0, 2 * np.sqrt(0.5) - 0.01), (c, 0, s, 0), (1, 1, 1))
    c = hull_hull(a, b)
    assert c.kind == "edge" and c.separation == pytest.approx(-0.01)


def test_tetrahedron_point_down():
    tet = tetra_half_edge_mesh()
    # turn the apex (vertex 3, above the base) to -z: a half turn about x; then lift the
    # hull so that the apex is 1 mm below the plane
    rot = (0.0, 1.0, 0.0, 0.0)
    lift = -pose_hull(tet, (0, 0, 0), rot, (1, 1, 1)).verts[:, 2].min() - 0.001
    h = pose_hull(tet, (0, 0, lift), rot, (1, 1, 1))
    c = hull_plane(h, UP, 0.0)
    # the most opposed face is a triangle through the apex; only the apex is below
    assert c.inc_size == 3 and c.below == 1
    assert hull_plane(pose_hull(tet, (0, 0, lift + 0.01), rot, (1, 1, 1)), UP, 0.0) is None


def test_octagon_on_octagon_at_yaw_pi_over_8():
    prism = ngon_prism_half_edge_mesh(8)
    pedestal = pose_hull(prism, (0, 0, 0.5), IDENTITY, (1, 1, 1))
    top = pose_hull(prism, (0, 0, 1.49), _yaw(np.pi / 8), (1, 1, 1))
    c = hull_hull(top, pedestal)
    assert c.kind == "face" and c.ref_size == 8 and c.inc_size == 8 and c.clipped == 16
    # and standing on the plane: an 8-point incident face
    p = hull_plane(top, UP, 0.99)
    assert p.inc_size == 8 and p.below == 8


def test_sphere_centre_inside_a_bipyramid():
    bip = pose_hull(bipyramid_half_edge_mesh(8), (1, 2, 3), _yaw(0.2), (1, 1, 1))
    assert sphere_hull((1.05, 2.0, 3.1), 0.3, bip) == "inside"
    assert sphere_hull((1.0, 2.0, 3.6 + 0.29), 0.3, bip) == "outside"     # above the apex
    assert sphere_hull((1.0, 2.0, 3.6 + 0.31), 0.3, bip) is None


# ---- what the goldens exercise ----------------------------------------------------------------

STATIC = {9, 10, 11}          # Plane, Wall, Pedestal
BIPYRAMID, DUMBBELL, CAPPED_BOX = 3, 7, 8
MARGIN = 0.01


def _classify(golden):
    """Counter of contact classes over every pair of every frame of a golden."""
    specs = hullpile_specs()
    W, steps, _, outs = load_golden(golden)
    pos, rot = outs["body_pos"].astype(np.float64), outs["body_rot"].astype(np.float64)
    scale, obj = outs["body_scale"].astype(np.float64), outs["body_object"]
    counts = Counter()
    bip_faces = set()
    for t in range(steps + 1):
        for w in range(W):
            prims = []           # (body, object, prim index, kind, posed, centre, reach)
            for b in range(pos.shape[2]):
                o = int(obj[t, w, b])
                for k, m in enumerate(specs[o]["prims"]):
                    if isinstance(m, dict):
                        h = pose_hull(m, pos[t, w, b], rot[t, w, b], scale[t, w, b])
                        c = h.verts.mean(axis=0)
                        prims.append((b, o, k, "hull", h, c, np.linalg.norm(h.verts - c, axis=1).max()))
                    elif m == "plane":
                        n = pose_hull(box_half_edge_mesh(), (0, 0, 0), rot[t, w, b], (1, 1, 1)).normals[1]
                        prims.append((b, o, k, "plane", (n, float(n @ pos[t, w, b])), None, None))
                    else:
                        r = m[1] * scale[t, w, b, 0]
                        prims.append((b, o, k, "sphere", r, pos[t, w, b], r))
            for i in range(len(prims)):
                for j in range(i + 1, len(prims)):
                    pa, pb = prims[i], prims[j]
                    if pa[0] == pb[0] or (pa[1] in STATIC and pb[1] in STATIC):
                        continue
                    if pa[3] == "plane" or (pa[3] == "sphere" and pb[3] == "hull"):
                        pa, pb = pb, pa
                    if pa[3] != "plane" and pb[3] != "plane" and \
                            np.linalg.norm(pa[5] - pb[5]) > pa[6] + pb[6] + MARGIN:
                        continue
                    touched = _classify_pair(pa, pb, counts, bip_faces, pos.shape[2])
                    for p in (pa, pb) if touched else ():
                        if p[1] in (DUMBBELL, CAPPED_BOX):
                            counts[("compound", p[1], p[2])] += 1
                    if touched and pa[1] in (DUMBBELL, CAPPED_BOX) and pb[1] in (DUMBBELL, CAPPED_BOX):
                        counts["compound-compound"] += 1
    counts["bipyramid faces"] = len(bip_faces)
    return counts


def _classify_pair(pa, pb, counts, bip_faces, bodies):
    if pa[3] == "hull" and pb[3] == "hull":
        c = hull_hull(pa[4], pb[4], MARGIN)
        if c is None:
            return False
        if c.kind == "edge":
            counts["edge-edge"] += 1
        else:
            counts["face"] += 1
            if c.ref_size == 8 and c.clipped > 8:
                counts["8-gon reference, >8 clipped"] += 1
            ref, inc = (pa, pb) if c.ref_is_a else (pb, pa)
            if ref[1] == BIPYRAMID:
                bip_faces.add(c.ref_face)
            if inc[1] == BIPYRAMID:
                bip_faces.add(c.inc_face)
        if BIPYRAMID in (pa[1], pb[1]):
            counts["bipyramid-hull"] += 1
        if max(pa[0], pb[0]) >= 48:
            counts["hull-hull at slot >= 48"] += 1
        return True
    if pa[3] == "hull" and pb[3] == "plane":
        c = hull_plane(pa[4], *pb[4], MARGIN)
        if c is None:
            return False
        counts["hull-plane"] += 1
        if c.inc_size == 8 and c.below == 8:
            counts["hull-plane 8-point face"] += 1
        if pa[1] == BIPYRAMID:
            bip_faces.add(c.inc_face)
        if pa[0] >= 48:
            counts["hull-plane at slot >= 48"] += 1
        return True
    if pa[3] == "hull" and pb[3] == "sphere":
        c = sphere_hull(pb[5], pb[4], pa[4], MARGIN)
        if c is None:
            return False
        counts["sphere-hull " + c] += 1
        return True
    return False              # sphere - sphere / sphere - plane: not the hull paths


@pytest.fixture(scope="module")
def pile_counts():
    return _classify("hullpile_w4_s150")


@pytest.fixture(scope="module")
def many_counts():
    return _classify("hullpile_many_w2_s100")


def test_golden_exercises_the_caps(pile_counts, many_counts):
    both = pile_counts + many_counts
    # A prism resting on the pedestal tilts by a few milliradians, and then an edge pair of
    # the two rims separates more than either face (the SAT path has no face bias): the
    # 8-gon face contacts come from landings, mostly in the 60-body variant's busier pile.
    assert both["8-gon reference, >8 clipped"] >= 20
    assert pile_counts["hull-plane 8-point face"] >= 100
    assert pile_counts["edge-edge"] >= 20
    assert pile_counts["bipyramid-hull"] >= 20
    assert pile_counts["bipyramid faces"] == 16
    assert pile_counts["sphere-hull inside"] >= 1 and pile_counts["sphere-hull outside"] >= 10
    for o in (DUMBBELL, CAPPED_BOX):
        for k in (0, 1):
            assert both[("compound", o, k)] >= 10, (o, k)
    assert both["compound-compound"] >= 1
    assert many_counts["hull-hull at slot >= 48"] >= 50
    assert many_counts["hull-plane at slot >= 48"] >= 50
