"""Lane-by-lane model of the XPBD solves' contact schedule (kernels_physics.cu): orderContacts,
which gives every contact of a world its dependency level, and sweepContactLevels, which runs
a warp's worlds level by level so that a parallel sweep reproduces the reference's sequential
Gauss-Seidel order.  Both are restated with the warp primitives the kernels use (ballots over
a group's lanes, group_shift, kGroupMask, __fns, __popc of the lower lanes), for LPW lanes per
world and 32 / LPW worlds per warp.  Also the float32 write-back of a static body, which
decides whether a static body may be left out of the ordering (bodySlotInfo).
Checked by tests/test_contact_schedule_model.py."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence, Tuple

import numpy as np

UNKNOWN_SLOT = 0x7FFF          # kUnknownSlot
MAX_LEVEL_BODIES = 128         # kMaxLevelBodies: the shared-memory level table
WARP = 32


def slot_info(slot: int, mutable: bool) -> int:
    """Contact::refInfo / altInfo: (world body slot << 1) | mutable (bodySlotInfo)."""
    s15 = UNKNOWN_SLOT if slot < 0 or slot >= UNKNOWN_SLOT else slot
    return (s15 << 1) | (1 if mutable else 0)


@dataclass
class World:
    """One world's candidates as orderContacts reads them: hit flag and the two body infos of
    every candidate slot, and its body count (num_slots comes from it)."""
    hits: Sequence[bool]
    ref_info: Sequence[int]
    alt_info: Sequence[int]
    bodies: int = 16


@dataclass
class Ordered:
    """What orderContacts writes for one world."""
    level: dict = field(default_factory=dict)      # candidate slot -> Contact::level
    order: List[int] = field(default_factory=list)  # contactOrder, candidate slots
    count: int = 0                                 # contactCounts
    max_level: int = 0                             # contactMaxLevel
    num_slots: int = MAX_LEVEL_BODIES


def group_mask(lpw: int) -> int:
    return 0xFFFFFFFF if lpw == 32 else (1 << lpw) - 1


def popc(x: int) -> int:
    return bin(x & 0xFFFFFFFF).count("1")


def ffs(x: int) -> int:
    """__ffs: 1 + index of the lowest set bit, 0 for none."""
    return (x & -x).bit_length() if x else 0


def fns(mask: int, base: int, offset: int) -> int:
    """__fns(mask, base, offset) for offset > 0: the offset-th set bit at or above base,
    0xffffffff when there is none."""
    assert offset > 0
    for b in range(base, 32):
        if (mask >> b) & 1:
            offset -= 1
            if offset == 0:
                return b
    return 0xFFFFFFFF


def num_slots_of(bodies: int, level_scratch: bool, max_world_bodies: int) -> int:
    """The level table orderContacts uses: the shared one of kMaxLevelBodies slots, or the
    world's row of PhysicsState::levelScratch when the world has more body slots."""
    if level_scratch and bodies > MAX_LEVEL_BODIES:
        return min(bodies, max_world_bodies)
    return MAX_LEVEL_BODIES


def order_contacts(world: World, lpw: int, level_scratch: bool = False, max_world_bodies: int = 128,
                   max_contacts: int = 1 << 30) -> Ordered:
    """orderContacts<LPW> for the LPW lanes of one world (the groups of a warp never exchange
    data in it: every ballot and shuffle is over the group's mask)."""
    gm = group_mask(lpw)
    num_slots = num_slots_of(world.bodies, level_scratch, max_world_bodies)
    last_level = [0] * num_slots
    n = len(world.hits)
    out = Ordered(num_slots=num_slots)
    running = max_level = seq_level = 0        # lane 0's registers (the scan)
    for base in range(0, n, lpw):
        hit = [base + sub < n and bool(world.hits[base + sub]) for sub in range(lpw)]
        a = [world.ref_info[base + sub] if hit[sub] else 0 for sub in range(lpw)]
        b = [world.alt_info[base + sub] if hit[sub] else 0 for sub in range(lpw)]
        hits = sum(1 << sub for sub in range(lpw) if hit[sub]) & gm       # ballot >> group_shift
        my_level = [0] * lpw
        todo = hits
        while todo:
            src = ffs(todo) - 1
            todo &= todo - 1
            sa_info, sb_info = a[src], b[src]                              # shuffles from src
            sa, sb = sa_info >> 1, sb_info >> 1
            if sa >= num_slots or sb >= num_slots:
                lvl = max_level + 1
                seq_level = lvl
            else:
                dep = seq_level
                if sa_info & 1:
                    dep = max(dep, last_level[sa])
                if sb_info & 1:
                    dep = max(dep, last_level[sb])
                lvl = dep + 1
                if sa_info & 1:
                    last_level[sa] = lvl
                if sb_info & 1:
                    last_level[sb] = lvl
            max_level = max(max_level, lvl)
            my_level[src] = lvl                                            # shuffle from lane 0
        for sub in range(lpw):
            if hit[sub]:
                i = base + sub
                at = running + popc(hits & ((1 << sub) - 1))
                out.level[i] = my_level[sub]
                if at < max_contacts:
                    while len(out.order) <= at:
                        out.order.append(-1)
                    out.order[at] = i
        running += popc(hits)
    out.count = min(running, max_contacts)
    out.max_level = max_level
    return out


def reference_levels(world: World, num_slots: int) -> dict:
    """Plain restatement of what the levels mean: in candidate order, a hit's level is one
    more than the deepest earlier hit it conflicts with (a shared mutable body slot, or a body
    of either outside the level table), 1 without one."""
    hits = [i for i, h in enumerate(world.hits) if h]
    level = {}
    for k, j in enumerate(hits):
        dep = 0
        for i in hits[:k]:
            if conflicts(world, i, j, num_slots):
                dep = max(dep, level[i])
        level[j] = dep + 1
    return level


def mutable_slots(world: World, i: int, num_slots: int) -> Tuple[set, bool]:
    """(mutable body slots of candidate i, whether it has a body outside the table)."""
    infos = (world.ref_info[i], world.alt_info[i])
    unknown = any((s >> 1) >= num_slots for s in infos)
    return {s >> 1 for s in infos if s & 1 and (s >> 1) < num_slots}, unknown


def conflicts(world: World, i: int, j: int, num_slots: int) -> bool:
    mi, ui = mutable_slots(world, i, num_slots)
    mj, uj = mutable_slots(world, j, num_slots)
    return ui or uj or bool(mi & mj)


def sweep_rounds(ordered: Sequence[Ordered], valid: Sequence[bool], lpw: int):
    """sweepContactLevels<LPW> over one warp: ordered[g] is what orderContacts left for the
    world of lane group g (valid[g] false: a group idling past the last world, n = levels = 0).
    Returns the rounds: per pair of __syncwarp()s, the (group, candidate slot, lane) of every
    solve the lanes run between them."""
    per_lane = WARP // lpw
    assert len(ordered) == per_lane and len(valid) == per_lane
    gm = group_mask(lpw)
    n = [o.count if v else 0 for o, v in zip(ordered, valid)]
    levels = [o.max_level if v else 0 for o, v in zip(ordered, valid)]
    # shfl_xor butterfly over o = LPW .. 16: every lane ends with the warp's maxima
    n_lane = [n[lane // lpw] for lane in range(WARP)]
    lv_lane = [levels[lane // lpw] for lane in range(WARP)]
    o = lpw
    while o < WARP:
        n_lane = [max(n_lane[l], n_lane[l ^ o]) for l in range(WARP)]
        lv_lane = [max(lv_lane[l], lv_lane[l ^ o]) for l in range(WARP)]
        o <<= 1
    assert len(set(n_lane)) == 1 and len(set(lv_lane)) == 1
    n_max, levels_max = n_lane[0], lv_lane[0]

    def contact_level(g, i):
        return ordered[g].level[ordered[g].order[i]]

    rounds = []
    for base in range(0, n_max, 32):
        lv = [[0] * per_lane for _ in range(WARP)]           # lv[lane][r]
        for lane in range(WARP):
            g, sub = lane // lpw, lane & (lpw - 1)
            for r in range(per_lane):
                i = base + r * lpw + sub
                lv[lane][r] = contact_level(g, i) if i < n[g] else 0
        for lvl in range(1, levels_max + 1):
            members = [0] * WARP
            for r in range(per_lane):
                ballot = sum(1 << lane for lane in range(WARP) if lv[lane][r] == lvl)
                for lane in range(WARP):
                    group_shift = (lane // lpw) * lpw
                    members[lane] |= ((ballot >> group_shift) & gm) << (r * lpw)
            solves = []
            for lane in range(WARP):
                g, sub = lane // lpw, lane & (lpw - 1)
                count = popc(members[lane])
                for k in range(sub, count, lpw):
                    m = fns(members[lane], 0, k + 1)
                    solves.append((g, ordered[g].order[base + m], lane))
            rounds.append(solves)
    return rounds


# ---- the write-back of a static body ----------------------------------------------------------
# Float32 restatement of what the solves do to a body whose inverse mass and inertia are 0
# (loadBodyMass of a static body): applyPositional's x and q updates and the velocity solve's
# v and o updates.

f32 = np.float32


def _cross(a, b):
    return (f32(a[1] * b[2]) - f32(a[2] * b[1]), f32(a[2] * b[0]) - f32(a[0] * b[2]),
            f32(a[0] * b[1]) - f32(a[1] * b[0]))


def rotate_vec(q, v):
    """Quat::rotateVec: v + 2 (w (q x v) + q x (q x v))."""
    w, qx, qy, qz = q
    qv = _cross((qx, qy, qz), v)
    qqv = _cross((qx, qy, qz), qv)
    return tuple(f32(v[k] + f32(f32(2) * f32(f32(qv[k] * w) + qqv[k]))) for k in range(3))


def quat_mul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (f32(f32(f32(aw * bw) - f32(ax * bx)) - f32(ay * by)) - f32(az * bz),
            f32(f32(f32(aw * bx) + f32(ax * bw)) + f32(ay * bz)) - f32(az * by),
            f32(f32(f32(aw * by) - f32(ax * bz)) + f32(ay * bw)) + f32(az * bx),
            f32(f32(f32(aw * bz) + f32(ax * by)) - f32(ay * bx)) + f32(az * bw))


def normalize(q):
    len2 = f32(f32(f32(q[0] * q[0]) + f32(q[1] * q[1])) + f32(q[2] * q[2])) + f32(q[3] * q[3])
    s = f32(f32(1) / np.sqrt(len2, dtype=f32))
    return tuple(f32(c * s) for c in q)


def angle_axis(angle, axis):
    c, s = np.cos(f32(angle) / f32(2), dtype=f32), np.sin(f32(angle) / f32(2), dtype=f32)
    return (f32(c), f32(axis[0] * s), f32(axis[1] * s), f32(axis[2] * s))


def positional_write_back(x, q, lam, n, tq, first: bool):
    """applyPositional for a static body as body 1 (first: x += ..., q += ...) or body 2
    (x -= ..., q -= ...): inv_m = 0, rot_axis = mulDiag(0, tq)."""
    x, q, lam = tuple(f32(c) for c in x), tuple(f32(c) for c in q), f32(lam)
    inv_m = f32(0)
    ra = tuple(f32(f32(0) * f32(t)) for t in tq)
    dx = tuple(f32(f32(lam * inv_m) * f32(c)) for c in n)
    half = f32(f32(0.5) * lam)
    w = rotate_vec(q, tuple(f32(half * c) for c in ra))
    dq = quat_mul((f32(0),) + w, q)
    if first:
        x = tuple(f32(a + d) for a, d in zip(x, dx))
        q = tuple(f32(a + d) for a, d in zip(q, dq))
    else:
        x = tuple(f32(a - d) for a, d in zip(x, dx))
        q = tuple(f32(a - d) for a, d in zip(q, dq))
    return x, normalize(q)


def velocity_write_back(v, o, q, impulse, n, ra_t, first: bool):
    """The velocity solve's update of a static body: v +-= n * impulse * 0, o +-= rotateVec of
    impulse * mulDiag(0, tq)."""
    v, o, impulse = tuple(f32(c) for c in v), tuple(f32(c) for c in o), f32(impulse)
    ra = tuple(f32(f32(0) * f32(t)) for t in ra_t)
    dv = tuple(f32(f32(f32(c) * impulse) * f32(0)) for c in n)
    do = rotate_vec(tuple(f32(c) for c in q), tuple(f32(impulse * c) for c in ra))
    sign = 1 if first else -1
    v = tuple(f32(a + d) if sign > 0 else f32(a - d) for a, d in zip(v, dv))
    o = tuple(f32(a + d) if sign > 0 else f32(a - d) for a, d in zip(o, do))
    return v, o


def set_velocity_of_unmoved(x, prev_x, h):
    """rowSetVelocity's linear velocity (x - prev.x) / h; the angular one is 2 / h * (0, 0, 0)
    when q equals prev.q under float ==."""
    lin = tuple(f32(f32(f32(a) - f32(b)) / f32(h)) for a, b in zip(x, prev_x))
    ang = tuple(f32(f32(f32(2) / f32(h)) * f32(0)) for _ in range(3))
    return lin, ang


def is_negative_zero(c) -> bool:
    return float(c) == 0.0 and bool(np.signbit(f32(c)))


def rotation_is_normalize_fixpoint(q) -> bool:
    n = normalize(q)
    return all(a == b for a, b in zip(n, (f32(c) for c in q)))


def static_is_mutable(x, q) -> bool:
    """bodySlotInfo's rule for a static body: it takes part in the ordering unless its
    rotation is a normalize fixpoint and none of its position and rotation components is -0."""
    if any(is_negative_zero(c) for c in tuple(x) + tuple(q)):
        return True
    return not rotation_is_normalize_fixpoint(q)


def bits(t) -> Tuple[int, ...]:
    return tuple(int(np.asarray(f32(c)).view(np.uint32)) for c in t)
