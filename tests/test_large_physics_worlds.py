"""Worlds of more than 128 rigid bodies, accepted with MADRONA_B200_MAX_BODIES_PER_WORLD: the
crowd simulator (sims/crowd: 20 to 1500 bodies per world, a different size every episode),
GPU engine vs the reference CPU backend.  Same bar as the other physics fixtures: every
exported column BIT-EXACT (1e-4 only with MADRONA_B200_FAST_MATH=1).  Worlds of up to 128
leaves take the warp-per-world candidate search, larger ones physFindCandidatesLargeKernel
(one block per world) in the same step, and the contact levels of worlds with more than
128 body slots live in a global table; neither changes a bit of the result.  Further cases
sit on the edges of that block search: a last leaf tile exactly full or of one leaf, the
4096-body cap, more large worlds than its persistent grid has blocks, and a second body
archetype (the crowd2 build variant)."""
import json
import os
import re

import numpy as np
import pytest

from oracle import runner
from sims import SIMS
from trace_utils import GOLDEN_DIR, assert_traces_equal, load_golden, rollout_gpu, trace_digests

EXACT = os.environ.get("MADRONA_B200_FAST_MATH", "0") != "1"
KNOB = "MADRONA_B200_MAX_BODIES_PER_WORLD"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _engine_constant(path, name):
    src = open(os.path.join(ROOT, "madrona_b200", "csrc", path)).read()
    m = re.search(r"constexpr int " + name + r" = (\d+);", src)
    assert m, name
    return int(m.group(1))


# leaves per shared-memory tile of physFindCandidatesLargeKernel, bodies per block chunk, and
# the largest knob value
SEARCH_TILE = _engine_constant("kernels_physics.cu", "kLargeSearchTile")
SEARCH_CHUNK = _engine_constant("kernels_physics.cu", "kLargeSearchThreads")
MAX_WORLD_BODIES = _engine_constant("physics_state.h", "kMaxWorldBodiesCap")
# room for the fixture's largest worlds: 1500 bodies, twice that while a respawn waits for
# compaction, their BVHs in the persistent arena, their candidates and contacts
CROWD_ENV = {"MADRONA_B200_ROWS_PER_WORLD": "3072", "MADRONA_B200_PERSIST_BYTES": str(512 << 20),
             "MADRONA_B200_MAX_CANDIDATES_PER_WORLD": "16384", "MADRONA_B200_MAX_CONTACTS_PER_WORLD": "8192"}

# golden name -> (worlds, steps, cfg); written by tests/golden/make_crowd_golden.py.  Seed 1:
# 128, 300 and 20 bodies over three episodes (the digests below hold the larger worlds)
CROWD_GOLDENS = {
    "crowd_w1_s30": (1, 30, {"seed": 1, "episode_len": 10}),
}
# Roll-outs kept as one SHA-256 per column of the reference CPU backend's trace.  One episode
# (episode_len 0): the handles of respawned bodies come from one pool for all worlds, handed
# out in another order by each backend, and a pair's order follows its entity IDs.
# name -> (sim, worlds, steps, cfg)
CROWD_REFERENCE_CASES = {
    # the 32 seeds give worlds of every size of the fixture, 20 to 1500 bodies
    "crowd_w32_s120": ("crowd", 32, 120, {"seed": 100, "episode_len": 0}),
    # every world at one size (uniform_bodies, plane and walls included: the world's leaves):
    # a last leaf tile exactly full (512, 1024) or of one leaf (513, 1025), and the knob's cap
    # (4096: eight full tiles).  By step 40 the bodies fly at up to 130 m/s
    "crowd_b512_w1_s40": ("crowd", 1, 40, {"seed": 1, "episode_len": 0, "uniform_bodies": 512}),
    "crowd_b513_w1_s40": ("crowd", 1, 40, {"seed": 1, "episode_len": 0, "uniform_bodies": 513}),
    "crowd_b1024_w1_s40": ("crowd", 1, 40, {"seed": 1, "episode_len": 0, "uniform_bodies": 1024}),
    "crowd_b1025_w1_s40": ("crowd", 1, 40, {"seed": 1, "episode_len": 0, "uniform_bodies": 1025}),
    "crowd_b4096_w2_s40": ("crowd", 2, 40, {"seed": 1, "episode_len": 0, "uniform_bodies": 4096}),
    # more large worlds than the block search's persistent grid holds (at most 8 blocks of 256
    # threads per SM): blocks take a second world and reuse their shared tile and scan sums
    "crowd_b129_w1100_s30": ("crowd", 1100, 30, {"seed": 500, "episode_len": 0, "uniform_bodies": 129}),
    # two body archetypes (crowd2: dynamic body i is a Body2 when i % 4 == 3): 905 Bodies and
    # 300 Body2s, each past one 256-body chunk with a partial last one, the Body2 slots 905 to
    # 1204, over three tiles; and 302 + 98 bodies in one tile, staged once for both archetypes
    "crowd2_b1205_w2_s40": ("crowd2", 2, 40, {"seed": 1, "episode_len": 0, "uniform_bodies": 1205}),
    "crowd2_b400_w1_s40": ("crowd2", 1, 40, {"seed": 1, "episode_len": 0, "uniform_bodies": 400}),
}
EDGE_CASES = [c for c in CROWD_REFERENCE_CASES if c != "crowd_w32_s120"]
TICKET_CASE = "crowd_b129_w1100_s30"
CROWD_DIGESTS_PATH = os.path.join(GOLDEN_DIR, "crowd_digests.json")

# sims/crowd: body j of a world is the plane (0), a wall (1 - 4) or kKinds[(j - 5) % 5]
KINDS = ("box", "ball", "wedge", "penta", "ball")
BALL_R = 0.5            # sims/objects.py hullpile_specs, scaled by 0.8 - 1.1


def _set_env(monkeypatch, knob="2048"):
    for k, v in CROWD_ENV.items():
        monkeypatch.setenv(k, v)
    if knob is not None:
        monkeypatch.setenv(KNOB, knob)


def _uniform_env(bodies):
    """Knobs for worlds of one size, `bodies` leaves each, with no respawn: the body tables never
    hold more than a world's bodies, and the knob is exactly the world's size, the largest world
    it accepts.  Counted on the reference's trace with each body as its bounding sphere grown
    by its motion, against slot boxes that only grow until the next rebuild, the fixture's
    worlds have at most about 4 candidate pairs per body by step 40 (16400 at 4096 bodies): 16
    per body leave four times that.  A contact is a candidate that hit: 8 per body leave twice
    that"""
    return {"MADRONA_B200_ROWS_PER_WORLD": str(bodies), "MADRONA_B200_PERSIST_BYTES": str(512 << 20),
            "MADRONA_B200_MAX_CANDIDATES_PER_WORLD": str(16 * bodies),
            "MADRONA_B200_MAX_CONTACTS_PER_WORLD": str(8 * bodies), KNOB: str(bodies)}


def _set_case_env(monkeypatch, case):
    bodies = CROWD_REFERENCE_CASES[case][3].get("uniform_bodies", 0)
    if not bodies:
        _set_env(monkeypatch)
        return
    for k, v in _uniform_env(bodies).items():
        monkeypatch.setenv(k, v)


def _run_until_error(ex, graph, steps):
    import madrona_b200 as mb
    for t in range(steps):
        try:
            ex.run(graph)
        except mb.MadronaB200Error as e:
            return t, str(e)
    return None, ""


def _device_still_healthy():
    import torch
    torch.cuda.synchronize()
    x = torch.arange(1024, device="cuda").sum().item()
    assert x == 1023 * 512


def _assert_matches_digests(case, got):
    sim, W, steps, cfg = CROWD_REFERENCE_CASES[case]
    if not EXACT:
        if not runner.available(sim):
            pytest.skip("a tolerance comparison needs the reference CPU backend (oracle/_ref)")
        ref, _ = runner.run_reference(SIMS[sim], W, steps, {}, cfg, workers=4)
        for k, w in ref.items():
            if isinstance(w, list):
                for g, r in zip(got[k], w):
                    if np.issubdtype(r.dtype, np.floating):
                        np.testing.assert_allclose(g, r, rtol=1e-4, atol=1e-5, err_msg=k)
                    else:
                        assert np.array_equal(g, r), k
            else:
                assert_traces_equal({k: got[k]}, {k: w})
        return
    with open(CROWD_DIGESTS_PATH) as f:
        want = json.load(f)[case]
    have = trace_digests(got)
    assert sorted(have) == sorted(want)
    differ = [k for k in sorted(want) if have[k] != want[k]]
    assert not differ, f"{case}: columns differ from the reference CPU backend: {differ}"


def _assert_close(got, outs):
    if EXACT:
        assert_traces_equal(got, outs)
        return
    for k, w in outs.items():
        if isinstance(w, list):
            assert len(got[k]) == len(w), k
            for g, r in zip(got[k], w):
                assert g.shape == r.shape, k
                if np.issubdtype(r.dtype, np.floating):
                    np.testing.assert_allclose(g, r, rtol=1e-4, atol=1e-5, err_msg=k)
                else:
                    assert np.array_equal(g, r), k
        else:
            assert_traces_equal({k: got[k]}, {k: w})


# ---- the golden itself (no GPU) --------------------------------------------------------------

def _world_rows(outs, t):
    """Per world of frame t: (positions, velocities) of its bodies, in world body order."""
    counts = outs["body_count"][t][:, 0]
    offs = np.concatenate([[0], np.cumsum(counts)])
    pos, vel = outs["body_pos"][t], outs["body_vel"][t]
    return [(pos[offs[w]:offs[w + 1]], vel[offs[w]:offs[w + 1]]) for w in range(len(counts))]


def test_golden_covers_both_search_paths():
    W, steps, _, outs = load_golden("crowd_w1_s30")
    counts = outs["body_count"][:, :, 0]
    assert counts.shape == (steps + 1, W)
    for t in range(steps + 1):
        assert len(outs["body_pos"][t]) == counts[t].sum()
    assert (counts > 128).any() and (counts <= 128).any()
    # a world crosses 128 bodies between episodes, both ways
    above = counts > 128
    assert (above[1:] & ~above[:-1]).any() and (~above[1:] & above[:-1]).any()


def test_golden_has_every_pair_class_in_contact():
    W, steps, _, outs = load_golden("crowd_w1_s30")
    seen = set()
    for t in range(1, steps + 1):
        for pos, vel in _world_rows(outs, t):
            n = len(pos)
            side = int(np.ceil(np.sqrt(n - 5)))
            pen = float(side)                  # the walls' inner faces (2 m per cell)
            kinds = np.array(["plane"] + ["wall"] * 4 + [KINDS[j % 5] for j in range(n - 5)])
            ball = kinds == "ball"
            hull = np.isin(kinds, ("box", "wedge", "penta"))
            bp = pos[ball]
            # two balls closer than two of the smallest radius: sphere - sphere
            if len(bp) > 1:
                d = np.linalg.norm(bp[:, None] - bp[None], axis=-1) + np.eye(len(bp)) * 1e9
                if (d < 2 * 0.8 * BALL_R).any():
                    seen.add("sphere-sphere")
            # resting on the floor: sphere - plane / hull - plane
            rest = np.abs(vel[:, 2]) < 0.05
            if (ball & ((rest & (pos[:, 2] < 1.1 * BALL_R + 0.01)) | (pos[:, 2] < 0.8 * BALL_R))).any():
                seen.add("sphere-plane")
            if (hull & rest & (pos[:, 2] < 0.6)).any():
                seen.add("hull-plane")
            # against a wall (a static box): sphere - hull / hull - hull
            reach = np.abs(pos[:, :2]).max(axis=1)
            if (ball & (reach > pen - 1.1 * BALL_R)).any():
                seen.add("sphere-hull")
            if (hull & (reach > pen - 0.3)).any():
                seen.add("hull-hull")
    assert seen == {"sphere-sphere", "sphere-plane", "hull-plane", "sphere-hull", "hull-hull"}, seen


@pytest.mark.skipif(not runner.available("crowd"), reason="oracle/_ref not built")
def test_reference_backend_reproduces_golden():
    W, steps, cfg = CROWD_GOLDENS["crowd_w1_s30"]
    _, _, _, outs = load_golden("crowd_w1_s30")
    got, _ = runner.run_reference(SIMS["crowd"], W, steps, {}, cfg, workers=1)
    assert_traces_equal(got, outs)


@pytest.mark.skipif(not runner.available("crowd"), reason="oracle/_ref not built")
def test_reference_backend_reproduces_digests():
    _, W, steps, cfg = CROWD_REFERENCE_CASES["crowd_w32_s120"]
    got, _ = runner.run_reference(SIMS["crowd"], W, steps, {}, cfg, workers=1)
    with open(CROWD_DIGESTS_PATH) as f:
        want = json.load(f)["crowd_w32_s120"]
    assert trace_digests(got) == want
    counts = got["body_count"][:, :, 0]
    assert (counts > 128).any() and (counts <= 128).any()


@pytest.mark.parametrize("case", EDGE_CASES)
def test_reference_backend_reproduces_edge_digests(case):
    sim, W, steps, cfg = CROWD_REFERENCE_CASES[case]
    if not runner.available(sim):
        pytest.skip("oracle/_ref not built")
    # the digests do not depend on the worker count (make_crowd_golden.py checks two)
    got, _ = runner.run_reference(SIMS[sim], W, steps, {}, cfg, workers=4)
    with open(CROWD_DIGESTS_PATH) as f:
        want = json.load(f)[case]
    assert trace_digests(got) == want
    # every world keeps its size for the whole roll-out
    assert (got["body_count"][:, :, 0] == cfg["uniform_bodies"]).all()


# ---- the case table reaches the edges it claims (no GPU) ----------------------------------------

# uniform-size case -> (leaf tiles, leaves in the last tile)
TILE_EDGES = {
    "crowd_b512_w1_s40": (1, 512),       # one tile, exactly full: staged once for all chunks
    "crowd_b513_w1_s40": (2, 1),         # a last tile of one leaf
    "crowd_b1024_w1_s40": (2, 512),      # two full tiles
    "crowd_b1025_w1_s40": (3, 1),
    "crowd_b4096_w2_s40": (8, 512),      # the knob's cap
}


def test_tile_cases_sit_on_the_tile_edges():
    assert SEARCH_TILE == 512 and MAX_WORLD_BODIES == 4096
    for case, (tiles, last) in TILE_EDGES.items():
        sim, W, steps, cfg = CROWD_REFERENCE_CASES[case]
        n = cfg["uniform_bodies"]
        assert -(-n // SEARCH_TILE) == tiles and n - SEARCH_TILE * (tiles - 1) == last, case
        assert sim == "crowd" and 1 <= W <= 2 and cfg["episode_len"] == 0, case
    sizes = sorted(CROWD_REFERENCE_CASES[c][3]["uniform_bodies"] for c in TILE_EDGES)
    assert sizes == [SEARCH_TILE, SEARCH_TILE + 1, 2 * SEARCH_TILE, 2 * SEARCH_TILE + 1, MAX_WORLD_BODIES]


def test_ticket_case_outnumbers_any_grid():
    # an SM holds at most 2048 threads, 8 search blocks, and an H100 SXM has 132 SMs; the GPU
    # test checks the device it runs on
    sim, W, steps, cfg = CROWD_REFERENCE_CASES[TICKET_CASE]
    assert cfg["uniform_bodies"] == 129 and W > 2048 // SEARCH_CHUNK * 132


@pytest.mark.parametrize("case", ["crowd2_b1205_w2_s40", "crowd2_b400_w1_s40"])
def test_two_archetype_cases_reach_the_chunk_and_slot_edges(case):
    sim, W, steps, cfg = CROWD_REFERENCE_CASES[case]
    if not runner.available(sim):
        pytest.skip("oracle/_ref not built")
    got, _ = runner.run_reference(SIMS[sim], W, 0, {}, cfg, workers=1)
    total, second = got["body_count"][0, :, 0], got["body_count"][0, :, 1]
    first = total - second
    assert len(got["body_pos"][0]) == first.sum() and len(got["body2_pos"][0]) == second.sum()
    assert (total == cfg["uniform_bodies"]).all()
    # Body takes slots [0, first), Body2 [first, total): Body2 slots past 128 and 256, and
    # Body past one block chunk with a partial last one
    assert (first > SEARCH_CHUNK).all() and (first % SEARCH_CHUNK != 0).all()
    if case == "crowd2_b1205_w2_s40":
        assert (first == 905).all() and (second == 300).all()
        assert (second > SEARCH_CHUNK).all() and (second % SEARCH_CHUNK != 0).all()
        assert (total > 2 * SEARCH_TILE).all()
    else:
        assert (first == 302).all() and (second == 98).all()
        assert (total <= SEARCH_TILE).all()


# ---- GPU: bit-exact against the reference ------------------------------------------------------

@pytest.mark.gpu
def test_gpu_matches_golden(monkeypatch):
    _set_env(monkeypatch)
    W, steps, cfg = CROWD_GOLDENS["crowd_w1_s30"]
    _, _, _, outs = load_golden("crowd_w1_s30")
    got, n_kernels = rollout_gpu("crowd", W, steps, None, cfg)
    assert n_kernels > 10
    _assert_close(got, outs)


@pytest.mark.gpu
@pytest.mark.parametrize("case,branches",
                         [pytest.param("crowd_w32_s120", None, id="graph_branches"),
                          pytest.param("crowd_w32_s120", "0", id="no_graph_branches")] +
                         [pytest.param(c, None, id=c) for c in EDGE_CASES])
def test_gpu_matches_reference_many_worlds(monkeypatch, case, branches):
    import torch
    _set_case_env(monkeypatch, case)
    if branches is not None:
        monkeypatch.setenv("MADRONA_B200_GRAPH_BRANCHES", branches)
    sim, W, steps, cfg = CROWD_REFERENCE_CASES[case]
    if case == TICKET_CASE:
        props = torch.cuda.get_device_properties(0)
        assert W > props.max_threads_per_multi_processor // SEARCH_CHUNK * props.multi_processor_count
    got, _ = rollout_gpu(sim, W, steps, None, cfg)
    _assert_matches_digests(case, got)


# ---- GPU: nothing changes for small worlds ----------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("sim,golden,cfg", [("room", "room_w4_s210", {"episode_len": 100, "seed": 21}),
                                            ("balls_many", "balls_many_w2_s60", {"seed": 9})])
def test_small_worlds_are_unchanged_by_the_knob(monkeypatch, sim, golden, cfg):
    if sim == "balls_many":     # 95 bodies: more rows and pairs than the defaults allow for
        for k, v in {"MADRONA_B200_MAX_CANDIDATES_PER_WORLD": "4096", "MADRONA_B200_MAX_CONTACTS_PER_WORLD": "2048",
                     "MADRONA_B200_ROWS_PER_WORLD": "128"}.items():
            monkeypatch.setenv(k, v)
    W, steps, ins, outs = load_golden(golden)
    plain, plain_kernels = rollout_gpu(sim, W, steps, ins or None, cfg)
    monkeypatch.setenv(KNOB, "4096")
    got, n_kernels = rollout_gpu(sim, W, steps, ins or None, cfg)
    # the large-world search is one more launch per step, and finds no world to search
    assert n_kernels == plain_kernels + 1
    for k, v in plain.items():
        assert np.array_equal(np.ascontiguousarray(got[k]).view(np.uint8),
                              np.ascontiguousarray(v).view(np.uint8)), k


@pytest.mark.gpu
def test_room_kernel_count_without_the_knob(monkeypatch):
    # bench.py's flagship, room at 8192 worlds, captures the 44 kernels it captured before
    from sims import make_executor
    monkeypatch.delenv(KNOB, raising=False)
    ex = make_executor("room", 8192, episode_len=100, seed=21)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    assert graph.num_kernels == 44
    del graph
    ex.close()


# ---- GPU: cliffs --------------------------------------------------------------------------------

@pytest.mark.gpu
def test_world_past_the_knob_raises(monkeypatch):
    # room for 256 bodies, a world of 300
    from sims import make_executor
    _set_env(monkeypatch, "256")
    ex = make_executor("crowd", 2, uniform_bodies=300, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 2)
    assert step == 0 and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
def test_world_one_past_the_knob_raises(monkeypatch):
    # room for 1024 bodies, a world of 1025: one leaf past the knob.  The world of exactly
    # 1024 bodies at a knob of 1024 runs and matches the reference (crowd_b1024_w1_s40 in
    # test_gpu_matches_reference_many_worlds)
    from sims import make_executor
    _set_env(monkeypatch, "1024")
    ex = make_executor("crowd", 2, uniform_bodies=1025, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 2)
    assert step == 0 and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
def test_large_world_past_the_candidate_cap_raises(monkeypatch):
    # 600 bodies on the block search with room for 512 candidates: once the 595 dynamic bodies
    # have landed, their plane pairs alone are more.  The world's candidates first pass 512 at
    # step 4 (and 1024 at step 9): it must raise there, after steps that match a run with room
    # to spare bit for bit, and leave the device usable
    import madrona_b200 as mb
    from sims import make_executor
    bodies, steps = 600, 40

    def run(cap):
        for k, v in _uniform_env(bodies).items():
            monkeypatch.setenv(k, v)
        monkeypatch.setenv("MADRONA_B200_MAX_CANDIDATES_PER_WORLD", str(cap))
        ex = make_executor("crowd", 1, uniform_bodies=bodies, seed=1, episode_len=0)
        graph = ex.buildLaunchGraphAllTaskGraphs()
        frames, step, msg = [], None, ""
        for t in range(steps):
            rows = ex.exportedNumRows(0)
            frames.append(ex.tensor(0, "float32", (rows, 3)).cpu().numpy().copy())
            try:
                ex.run(graph)
            except mb.MadronaB200Error as e:
                step, msg = t, str(e)
                break
        _device_still_healthy()
        ex.close()
        return frames, step, msg

    capped, step, msg = run(512)
    assert step == 4 and "physics buffer overflow" in msg, (step, msg)
    roomy, clean_step, clean_msg = run(16 * bodies)
    assert clean_step is None, (clean_step, clean_msg)
    # frames 0 .. step: the state before each step up to the one that overflowed
    assert len(capped) == step + 1
    for t, (a, b) in enumerate(zip(capped, roomy)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), t


@pytest.mark.gpu
@pytest.mark.parametrize("value", ["127", "4097", "abc", "256x", ""])
def test_bad_knob_value_fails_executor_creation(monkeypatch, value):
    import madrona_b200 as mb
    from sims import make_executor
    monkeypatch.setenv(KNOB, value)
    with pytest.raises(mb.MadronaB200Error, match=KNOB):
        make_executor("balls", 4, seed=1)
    assert KNOB in mb.load_library().mb2_last_error().decode()
    _device_still_healthy()


@pytest.mark.gpu
def test_tree_too_deep_for_the_rebuild_raises(monkeypatch):
    # 100 bodies on a geometric spiral: the rebuild's stacks would need more than 64 entries
    from sims import make_executor
    _set_env(monkeypatch)
    ex = make_executor("crowd", 2, uniform_bodies=100, layout=1, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 2)
    assert step == 0 and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


# ---- GPU: snapshot ------------------------------------------------------------------------------

@pytest.mark.gpu
def test_snapshot_restore_with_large_worlds(monkeypatch):
    # the large-world list and the level table are per-step scratch: neither is part of a
    # snapshot, and "save, step, restore, step" repeats bit for bit, episode resets included
    from sims import make_executor
    _set_env(monkeypatch)
    W = 8
    ex = make_executor("crowd", W, seed=3, episode_len=15)
    graph = ex.buildLaunchGraphAllTaskGraphs()

    def read():
        rows = ex.exportedNumRows(0)
        cols = [ex.tensor(0, "float32", (rows, 3)), ex.tensor(1, "float32", (rows, 4)),
                ex.tensor(2, "float32", (rows, 6)), ex.tensor(3, "int32", (rows, 2)),
                ex.tensor(4, "int32", (W, 1))]
        return [c.cpu().numpy().copy() for c in cols]

    for _ in range(10):
        ex.run(graph)
    with ex.snapshot() as snap:
        snap.save()
        for _ in range(12):
            ex.run(graph)
        first = read()
        snap.restore()
        for _ in range(12):
            ex.run(graph)
        second = read()
    for a, b in zip(first, second):
        assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert (first[4] > 128).any()
    ex.close()
