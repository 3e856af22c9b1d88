"""Worlds of more than 128 rigid bodies, accepted with MADRONA_B200_MAX_BODIES_PER_WORLD: the
crowd simulator (sims/crowd: 20 to 1500 bodies per world, a different size every episode),
GPU engine vs the reference CPU backend.  Same bar as the other physics fixtures: every
exported column BIT-EXACT (1e-4 only with MADRONA_B200_FAST_MATH=1).  Worlds of up to 128
leaves take the warp-per-world candidate search, larger ones physFindCandidatesLargeKernel
(one block per world) in the same step, and the contact levels of worlds with more than
128 body slots live in a global table; neither changes a bit of the result."""
import json
import os

import numpy as np
import pytest

from oracle import runner
from sims import SIMS
from trace_utils import GOLDEN_DIR, assert_traces_equal, load_golden, rollout_gpu, trace_digests

EXACT = os.environ.get("MADRONA_B200_FAST_MATH", "0") != "1"
KNOB = "MADRONA_B200_MAX_BODIES_PER_WORLD"
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
# out in another order by each backend, and a pair's order follows its entity IDs; the 32
# seeds give worlds of every size of the fixture, 20 to 1500 bodies
CROWD_REFERENCE_CASES = {
    "crowd_w32_s120": (32, 120, {"seed": 100, "episode_len": 0}),
}
CROWD_DIGESTS_PATH = os.path.join(GOLDEN_DIR, "crowd_digests.json")

# sims/crowd: body j of a world is the plane (0), a wall (1 - 4) or kKinds[(j - 5) % 5]
KINDS = ("box", "ball", "wedge", "penta", "ball")
BALL_R = 0.5            # sims/objects.py hullpile_specs, scaled by 0.8 - 1.1


def _set_env(monkeypatch, knob="2048"):
    for k, v in CROWD_ENV.items():
        monkeypatch.setenv(k, v)
    if knob is not None:
        monkeypatch.setenv(KNOB, knob)


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
    W, steps, cfg = CROWD_REFERENCE_CASES[case]
    if not EXACT:
        if not runner.available("crowd"):
            pytest.skip("a tolerance comparison needs the reference CPU backend (oracle/_ref)")
        ref, _ = runner.run_reference(SIMS["crowd"], W, steps, {}, cfg, workers=1)
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
    W, steps, cfg = CROWD_REFERENCE_CASES["crowd_w32_s120"]
    got, _ = runner.run_reference(SIMS["crowd"], W, steps, {}, cfg, workers=1)
    with open(CROWD_DIGESTS_PATH) as f:
        want = json.load(f)["crowd_w32_s120"]
    assert trace_digests(got) == want
    counts = got["body_count"][:, :, 0]
    assert (counts > 128).any() and (counts <= 128).any()


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
@pytest.mark.parametrize("branches", [None, "0"], ids=["graph_branches", "no_graph_branches"])
def test_gpu_matches_reference_many_worlds(monkeypatch, branches):
    _set_env(monkeypatch)
    if branches is not None:
        monkeypatch.setenv("MADRONA_B200_GRAPH_BRANCHES", branches)
    W, steps, cfg = CROWD_REFERENCE_CASES["crowd_w32_s120"]
    got, _ = rollout_gpu("crowd", W, steps, None, cfg)
    _assert_matches_digests("crowd_w32_s120", got)


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
