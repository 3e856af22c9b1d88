"""The contact schedule of the XPBD solves (tests/contact_schedule_model.py restates
orderContacts and sweepContactLevels lane by lane) at 8, 16 and 32 lanes per world: every
contact of every valid world is solved exactly once and idle lane groups solve nothing; no
round (the solves between two __syncwarp()s) holds two contacts of one world that share a
mutable body slot or a body outside the level table; contacts that share a mutable slot are
solved in contactOrder's order, the reference's sequential order; contacts that share only a
static body are not serialized.  Inputs: contact counts around the lane and chunk edges, one
long chain, independent contacts, unknown slots, worlds past the shared level table (the
global levelScratch rows), warp-mates of very different depth, the last warp with 1 to 3
valid worlds, and seeded random worlds.  CPU only.

The static-body rule.  A static body is left out of the ordering on the premise that writing
it back is a no-op, so same-level writers cannot disagree.  In float32 the solves add exactly
+-0 to a static body's position and rotation (inverse mass and inertia 0), and x + (+-0) == x
bit for bit except for a stored -0: -0 + (+0) == +0 (and -0 - (-0) == +0).  Which sign the
zero has depends on the sign of lambda and of the contact normal, so two writers of one
static body at one level CAN disagree: with a component at -0, one writes +0, the other -0,
and the last to store wins, where the reference's sequential sweep always ends at +0.
Quat::angleAxis with a negative angle about z stores -0 in x and y, and such a rotation is a
normalize fixpoint.  So the rule was incomplete; bodySlotInfo now orders a static body that
has a -0 in its position or rotation like a dynamic one (a component the write-back turns
into +0 stays +0, so from the next step on the body is left out again).  Without a -0, the
position write-back is a bitwise no-op for either sign of lambda, as modelled below.  The
velocity solve's write-back (v -= n * impulse * 0, o -= rotateVec(impulse * 0)) is a no-op
too: rowSetVelocity leaves a static body's velocities at +0 ((x - prev.x) / h of an unmoved
or -0 -> +0 body is +0), and +0 + (+-0) == +0."""
import itertools
from collections import Counter

import numpy as np
import pytest

from contact_schedule_model import (MAX_LEVEL_BODIES, UNKNOWN_SLOT, World, angle_axis, bits, conflicts,
                                    fns, is_negative_zero, normalize, order_contacts, positional_write_back,
                                    reference_levels, rotation_is_normalize_fixpoint, set_velocity_of_unmoved,
                                    slot_info, static_is_mutable, sweep_rounds, velocity_write_back)

LANES = [8, 16, 32]
PLANE = 0                 # body slot of a static plane in the worlds below


def world_of(pairs, bodies=16, static=(PLANE,), misses=(), unknown=()):
    """Candidates (a, b) of body slots; slots in `static` are non-mutable, slots in `unknown`
    are written as kUnknownSlot; candidates listed in `misses` are not hits."""
    def info(s):
        return slot_info(UNKNOWN_SLOT if s in unknown else s, s not in static)
    return World(hits=[i not in misses for i in range(len(pairs))],
                 ref_info=[info(a) for a, _ in pairs], alt_info=[info(b) for _, b in pairs], bodies=bodies)


def random_world(rng, n, bodies=16, p_miss=0.2, p_plane=0.3, p_unknown=0.0):
    pairs, unknown = [], set()
    for _ in range(n):
        a = PLANE if rng.random() < p_plane else int(rng.integers(1, bodies))
        b = int(rng.integers(1, bodies))
        pairs.append((a, b))
    if p_unknown:
        unknown = {int(s) for s in rng.integers(1, bodies, size=2)} if rng.random() < p_unknown else set()
    misses = {i for i in range(n) if rng.random() < p_miss}
    return world_of(pairs, bodies, misses=misses, unknown=unknown)


def check_warp(worlds, valid, lpw, level_scratch=False, max_world_bodies=128):
    """Runs one warp of the schedule and checks it; returns (ordered, rounds)."""
    ordered = [order_contacts(w, lpw, level_scratch, max_world_bodies) for w in worlds]
    for w, o, v in zip(worlds, ordered, valid):
        if not v:
            continue
        hits = [i for i, h in enumerate(w.hits) if h]
        assert o.order == hits and o.count == len(hits)
        assert o.level == reference_levels(w, o.num_slots)
        assert o.max_level == max(o.level.values(), default=0)
    rounds = sweep_rounds(ordered, valid, lpw)

    solved = Counter((g, i) for r in rounds for g, i, _ in r)
    want = Counter((g, i) for g, o in enumerate(ordered) if valid[g] for i in o.order)
    assert solved == want                               # exactly once; idle groups solve nothing
    round_of = {(g, i): k for k, r in enumerate(rounds) for g, i, _ in r}
    for r in rounds:
        for g, i, lane in r:
            assert lane // lpw == g                     # a world's contacts run on its own lanes
        for (g1, i1, _), (g2, i2, _) in itertools.combinations(r, 2):
            if g1 == g2:
                assert not conflicts(worlds[g1], i1, i2, ordered[g1].num_slots), (g1, i1, i2)
    for g, o in enumerate(ordered):
        if not valid[g]:
            continue
        for x, y in itertools.combinations(range(o.count), 2):
            i, j = o.order[x], o.order[y]
            if conflicts(worlds[g], i, j, o.num_slots):
                assert round_of[(g, i)] < round_of[(g, j)], (g, i, j)
    return ordered, rounds


def check_alone(world, lpw, **kw):
    per = 32 // lpw
    return check_warp([world] * per, [True] + [False] * (per - 1), lpw, **kw)


# ---- the warp primitives ---------------------------------------------------------------------

def test_fns_finds_the_nth_set_bit():
    assert fns(0b10110, 0, 1) == 1 and fns(0b10110, 0, 2) == 2 and fns(0b10110, 0, 3) == 4
    assert fns(0b10110, 0, 4) == 0xFFFFFFFF
    assert fns(0x80000000, 0, 1) == 31


# ---- orderContacts + sweepContactLevels ----------------------------------------------------

@pytest.mark.parametrize("lpw", LANES)
def test_contact_counts_around_the_lane_and_chunk_edges(lpw):
    rng = np.random.default_rng(1000 + lpw)
    for n in sorted({0, 1, lpw - 1, lpw, lpw + 1, 31, 32, 33, 64, 65, 300}):
        check_alone(random_world(rng, n), lpw)
        per = 32 // lpw
        check_warp([random_world(rng, n) for _ in range(per)], [True] * per, lpw)


@pytest.mark.parametrize("lpw", LANES)
@pytest.mark.parametrize("n", [33, 100, 300])
def test_one_long_chain(lpw, n):
    # every contact on body 1: n levels, one contact per round, in candidate order
    w = world_of([(1, 1 + (k % 2)) if k % 3 else (PLANE, 1) for k in range(n)])
    ordered, rounds = check_alone(w, lpw)
    assert ordered[0].max_level == n
    assert [i for r in rounds for _, i, _ in r] == list(range(n))


@pytest.mark.parametrize("lpw", LANES)
def test_independent_contacts_are_one_level(lpw):
    w = world_of([(2 * k + 1, 2 * k + 2) for k in range(60)], bodies=121)
    ordered, rounds = check_alone(w, lpw)
    assert ordered[0].max_level == 1
    assert len([r for r in rounds if r]) == 2          # two chunks of 32, one level each


@pytest.mark.parametrize("lpw", LANES)
def test_a_plane_under_every_contact_is_not_serialized(lpw):
    # 40 bodies resting on one static plane (and a static wall): the levels stay flat
    pairs = [(PLANE, k) for k in range(1, 41)] + [(41, k) for k in range(1, 9)]
    w = world_of(pairs, bodies=42, static=(PLANE, 41))
    ordered, rounds = check_alone(w, lpw)
    levels = [ordered[0].level[i] for i in range(len(pairs))]
    assert levels == [1] * 40 + [2] * 8
    # the same world with a mutable plane is one chain
    chained = check_alone(world_of(pairs, bodies=42, static=()), lpw)[0]
    assert chained[0].max_level == 40


@pytest.mark.parametrize("lpw", LANES)
def test_unknown_slots_are_ordered_after_everything_before(lpw):
    rng = np.random.default_rng(7 + lpw)
    for n in (5, 40, 70):
        pairs = [(int(rng.integers(0, 8)), int(rng.integers(1, 8))) for _ in range(n)]
        w = world_of(pairs, bodies=8, unknown=(3,), misses=set(range(0, n, 7)))
        ordered, rounds = check_alone(w, lpw)
        lv = ordered[0].level
        for i in lv:
            if 3 in pairs[i]:
                # strictly after every earlier hit, strictly before every later one
                assert all(lv[j] < lv[i] for j in lv if j < i)
                assert all(lv[j] > lv[i] for j in lv if j > i)
                assert sum(1 for r in rounds for _, k, _ in r if k == i) == 1
                (r,) = [r for r in rounds if any(k == i for _, k, _ in r)]
                assert len(r) == 1


@pytest.mark.parametrize("lpw", LANES)
def test_world_past_the_shared_level_table(lpw):
    # 300 bodies: the levels live in the world's levelScratch row (num_slots = min(bodies,
    # maxWorldBodies)); slots past a smaller cap count as unknown
    rng = np.random.default_rng(300 + lpw)
    pairs = [(int(rng.integers(0, 300)), int(rng.integers(1, 300))) for _ in range(400)]
    pairs += [(k, 299) for k in range(130, 170)]                   # slots past 128 in a chain
    w = world_of(pairs, bodies=300)
    ordered, _ = check_alone(w, lpw, level_scratch=True, max_world_bodies=4096)
    assert ordered[0].num_slots == 300
    assert max(ordered[0].level[i] for i in range(400, 440)) >= 40
    capped, _ = check_alone(w, lpw, level_scratch=True, max_world_bodies=200)
    assert capped[0].num_slots == 200
    # without the table, the shared one (128 slots) treats every body past it as unknown
    shared, _ = check_alone(w, lpw, level_scratch=False)
    assert shared[0].num_slots == MAX_LEVEL_BODIES
    assert shared[0].max_level > capped[0].max_level > ordered[0].max_level


@pytest.mark.parametrize("lpw", [8, 16])
def test_warp_mates_of_very_different_depth(lpw):
    rng = np.random.default_rng(50 + lpw)
    per = 32 // lpw
    chain = world_of([(1, 2)] * 90)
    worlds = [chain, world_of([]), random_world(rng, 250, bodies=120), world_of([(k, k + 1) for k in range(1, 9)])]
    for perm in itertools.permutations(range(per)):
        ws = [worlds[p] for p in perm]
        ordered, _ = check_warp(ws, [True] * per, lpw)
        assert ordered[perm.index(0)].max_level == 90
        assert ordered[perm.index(1)].count == 0


@pytest.mark.parametrize("lpw", [8, 16])
def test_last_warp_with_idle_groups(lpw):
    # solverWorld: the groups past the last world idle along on it with valid = false
    rng = np.random.default_rng(90 + lpw)
    per = 32 // lpw
    for valid_worlds in range(1, per):
        for n in (0, 1, 33, 120):
            worlds = [random_world(rng, n) for _ in range(valid_worlds)]
            worlds += [worlds[-1]] * (per - valid_worlds)
            check_warp(worlds, [True] * valid_worlds + [False] * (per - valid_worlds), lpw)


@pytest.mark.parametrize("lpw", LANES)
def test_random_warps(lpw):
    rng = np.random.default_rng(2024 + lpw)
    per = 32 // lpw
    for _ in range(25):
        worlds = []
        for _ in range(per):
            n = int(rng.choice([0, 1, 5, 31, 32, 33, 70, 130, 260]))
            bodies = int(rng.choice([3, 16, 48, 128]))
            worlds.append(random_world(rng, n, bodies=bodies, p_miss=float(rng.random() * 0.5),
                                       p_plane=float(rng.random()), p_unknown=0.3))
        valid_worlds = int(rng.integers(1, per + 1))
        valid = [g < valid_worlds for g in range(per)]
        worlds = [w if v else worlds[valid_worlds - 1] for w, v in zip(worlds, valid)]
        check_warp(worlds, valid, lpw)


# ---- the static-body write-back ------------------------------------------------------------

NEG0, POS0 = np.float32(-0.0), np.float32(0.0)


def _normals(rng):
    out = [(0.0, 0.0, 1.0), (0.0, 0.0, -1.0), (1.0, 0.0, 0.0), (0.0, -1.0, 0.0)]
    for _ in range(6):
        v = rng.normal(size=3)
        out.append(tuple(v / np.linalg.norm(v)))
    return out


def _arms(rng):
    out = [(0.0, 0.0, 0.0), (-0.0, 0.0, -0.0), (1.0, -2.0, 0.5), (-1.0, 2.0, -0.5)]
    out += [tuple(rng.normal(size=3)) for _ in range(4)]
    return out


def _writes(x, q, rng):
    """Every write-back of body (x, q) by a contact: both sides, both signs of lambda."""
    out = []
    for lam, n, tq, first in itertools.product((0.37, -0.37, 1e-30, -2.5e3), _normals(rng), _arms(rng),
                                               (True, False)):
        out.append(positional_write_back(x, q, lam, n, tq, first))
    return out


def _fixpoints(rng):
    qs = [(1.0, 0.0, 0.0, 0.0), angle_axis(0.7, (0.0, 0.0, 1.0)), angle_axis(np.pi, (0.0, 0.0, 1.0))]
    while len(qs) < 12:
        v = rng.normal(size=4).astype(np.float32)
        q = normalize(tuple(v))
        if rotation_is_normalize_fixpoint(q):
            qs.append(q)
    return qs


def test_write_back_without_negative_zero_is_a_no_op():
    rng = np.random.default_rng(5)
    for q in _fixpoints(rng):
        assert rotation_is_normalize_fixpoint(q)
        q = tuple(abs(c) if c == 0 else c for c in q)            # no -0
        for x in [(0.0, 0.0, 0.0), (1.5, 0.0, -3.25), tuple(rng.normal(size=3) * 10)]:
            assert not static_is_mutable(x, q)
            for wx, wq in _writes(x, q, rng):
                assert bits(wx) == bits(x) and bits(wq) == bits(q)


def test_negative_zero_makes_same_level_writers_disagree():
    rng = np.random.default_rng(6)
    # a position component at -0: lambda > 0 adds +0 (-> +0), lambda < 0 adds -0 (stays -0)
    x, q = (1.0, NEG0, 2.0), (1.0, 0.0, 0.0, 0.0)
    up = (0.0, 1.0, 0.0)
    a, _ = positional_write_back(x, q, 0.5, up, (1.0, 1.0, 1.0), True)
    b, _ = positional_write_back(x, q, -0.5, up, (1.0, 1.0, 1.0), True)
    assert not is_negative_zero(a[1]) and is_negative_zero(b[1])
    # the sequential sweep ends at +0 in either order; a same-level race can end at -0
    for first, second in ((0.5, -0.5), (-0.5, 0.5)):
        y, _ = positional_write_back(x, q, first, up, (1.0, 1.0, 1.0), True)
        y, _ = positional_write_back(y, q, second, up, (1.0, 1.0, 1.0), True)
        assert not is_negative_zero(y[1])
    assert static_is_mutable(x, q)

    # angleAxis with a negative angle about z: q.x = q.y = -0, and a normalize fixpoint, so the
    # rotation-only rule would have left it out of the ordering
    yaw = angle_axis(-1.0, (0.0, 0.0, 1.0))
    assert is_negative_zero(yaw[1]) and is_negative_zero(yaw[2])
    assert rotation_is_normalize_fixpoint(yaw)
    results = {bits(wq) for _, wq in _writes((0.0, 0.0, 0.0), yaw, rng)}
    assert len(results) > 1
    assert static_is_mutable((0.0, 0.0, 0.0), yaw)


def test_the_rule_covers_every_write_back_that_changes_a_body():
    rng = np.random.default_rng(7)
    changed = 0
    for _ in range(40):
        q = _fixpoints(rng)[int(rng.integers(0, 12))]
        q = tuple(NEG0 if c == 0 and rng.random() < 0.5 else c for c in q)
        x = tuple(rng.choice([NEG0, POS0, np.float32(rng.normal())]) for _ in range(3))
        writes = _writes(x, q, rng)
        moved = any(bits(wx) != bits(x) or bits(wq) != bits(q) for wx, wq in writes)
        if not static_is_mutable(x, q):
            assert not moved, (x, q)
        changed += moved
    assert changed > 0


def test_velocity_write_back_of_a_static_body_is_a_no_op():
    rng = np.random.default_rng(8)
    h = 1.0 / 60 / 4
    for x, prev in [((1.0, 0.0, -2.0), (1.0, 0.0, -2.0)), ((POS0, NEG0, 3.0), (NEG0, NEG0, 3.0)),
                    ((NEG0, NEG0, NEG0), (NEG0, NEG0, NEG0))]:
        v, o = set_velocity_of_unmoved(x, prev, h)
        assert bits(v) == bits((POS0,) * 3) and bits(o) == bits((POS0,) * 3)
        for q in _fixpoints(rng)[:4] + [angle_axis(-0.4, (0.0, 0.0, 1.0))]:
            for impulse, n, ra, first in itertools.product((0.8, -0.8), _normals(rng), _arms(rng), (True, False)):
                wv, wo = velocity_write_back(v, o, q, impulse, n, ra, first)
                assert bits(wv) == bits(v) and bits(wo) == bits(o)
