"""Physics overlap queries: PhysicsSystem::findEntitiesWithinAABB,
checkEntityAABBOverlap and the standalone broadphase overlap tasks (CandidateCollision
rows without the solver), on sims/triggers (no solver) and sims/buttons (queries after
the XPBD step, on the refitted tree).  The reference CPU backend's traces are kept as
goldens (tests/golden/triggers_w3_s200.npz, buttons_w4_s220.npz) and as per-column
digests of larger roll-outs (tests/golden/overlap_digests.json), both written by
tests/golden/make_overlap_golden.py from the harnesses oracle/overlap.mk builds; where
those harnesses exist the GPU is also compared with live reference roll-outs."""
import json
import os

import numpy as np
import pytest

from sims.inputs import buttons_inputs, triggers_inputs
from trace_utils import GOLDEN_DIR, assert_traces_equal, load_golden, rollout_gpu, trace_digests

INPUTS = {"triggers": triggers_inputs, "buttons": buttons_inputs}
# golden file -> (sim, worlds, steps, sim cfg); inputs: INPUTS[sim](W, steps, seed=1234)
GOLDENS = {
    "triggers_w3_s200": ("triggers", 3, 200, {"seed": 11}),
    "buttons_w4_s220": ("buttons", 4, 220, {"episode_len": 100, "seed": 21}),
}
GOLDEN = ("triggers_w3_s200",) + GOLDENS["triggers_w3_s200"][1:]
# name -> (sim, worlds, steps, seed of the inputs, sim cfg)
OVERLAP_REFERENCE_CASES = {
    "triggers_w300_s150": ("triggers", 300, 150, 9, {"seed": 500}),
    "buttons_w200_s120": ("buttons", 200, 120, 5, {"episode_len": 60, "seed": 900}),
}
OVERLAP_DIGESTS_PATH = os.path.join(GOLDEN_DIR, "overlap_digests.json")
K_PAIRS = 32


def overlap_case(name):
    sim, W, steps, seed, cfg = OVERLAP_REFERENCE_CASES[name]
    return sim, W, steps, INPUTS[sim](W, steps, seed=seed), dict(cfg)


def _pairs(outs):
    """[steps + 1, W] counts and [steps + 1, W, K, 4] pairs (a id, b id, aPrim, bPrim)."""
    p = outs["pairs"]
    return p[..., 0], p[..., 1:].reshape(p.shape[0], p.shape[1], K_PAIRS, 4)


def _digests():
    with open(OVERLAP_DIGESTS_PATH) as f:
        return json.load(f)


# ---- CPU: the goldens exercise the feature -------------------------------------------------

def test_golden_pairs_vary_and_include_compound_primitives():
    W, steps, ins, outs = load_golden(GOLDEN[0])
    counts, pairs = _pairs(outs)
    assert counts[1:].min() > 0 and len(np.unique(counts)) > 3
    listed = pairs[..., 0] >= 0
    # the dumbbell's second hull shows up on either side of a pair
    assert ((pairs[..., 2] > 0) & listed).any() and ((pairs[..., 3] > 0) & listed).any()
    # side a is the body with the smaller entity ID
    assert (pairs[..., 0][listed] < pairs[..., 1][listed]).all()


def test_golden_has_no_static_static_pair_and_pickups_churn():
    W, steps, ins, outs = load_golden(GOLDEN[0])
    counts, pairs = _pairs(outs)
    ids = outs["pickup_entity"]
    # floor and the four walls are the first five props of each world (static)
    walls_floor = outs["prop_entity"][:, :, :5, 1]
    seen = set()
    for t in range(1, steps + 1):
        seen.update(map(tuple, ids[t].tolist()))     # (gen, id): IDs are recycled
        static = np.concatenate([ids[t][:, 1], walls_floor[t].ravel()])
        listed = pairs[t][..., 0] >= 0
        a = np.isin(pairs[t][..., 0], static) & listed
        b = np.isin(pairs[t][..., 1], static) & listed
        assert not (a & b).any(), f"static - static pair at step {t}"
        # every body of a world sits on the floor plane, so kinematic - floor pairs appear
        assert (np.isin(pairs[t][..., :2], walls_floor[t][:, 0]) & listed[..., None]).any()
    zone = outs["zone"]
    assert zone[-1, :, 6].min() > 0, "every world replaced pickups"
    assert len(seen) > W * 6


def test_golden_zone_queries_skip_the_sphere():
    W, steps, ins, outs = load_golden(GOLDEN[0])
    zone = outs["zone"]
    # the ball's centre crosses the zone, checkEntityAABBOverlap never reports it (sphere only)
    assert zone[..., 5].sum() > 0 and zone[..., 4].sum() == 0
    # the dumbbell (two hulls) is found in some steps and not in others
    assert 0 < zone[..., 3].sum() < zone[..., 3].size
    assert (zone[..., 0] > 0).any() and (zone[..., 0] == 0).any()


def test_buttons_golden_presses_opens_doors_and_skips_the_ball():
    W, steps, ins, outs = load_golden("buttons_w4_s220")
    state = outs["button_state"]            # [steps + 1, W, button, (pressed, found, first, ballOn)]
    pressed = state[1:, ..., 0]
    assert 0 < pressed.sum() < pressed.size, "buttons pressed in some steps, not in others"
    assert (np.diff(pressed, axis=0) != 0).any(), "a button is pressed and released again"
    # the doors follow their buttons: they sink and rise again
    door_z = outs["door_pos"][..., 2]
    assert door_z.min() < 0 < 1.0 == door_z.max()
    assert (np.diff(door_z, axis=0) < 0).any() and (np.diff(door_z, axis=0) > 0).any()
    # a ball on a button is not reported: with the ball's centre on button 1 and nothing
    # else reported, the button stays up (the sphere's leaf box overlaps the plate)
    ball_on = state[1:, :, 1, 3] == 1
    assert ball_on.sum() > steps and (pressed[:, :, 1][ball_on] == 0).sum() > steps
    assert (state[1:, :, 1, 1][ball_on & (pressed[:, :, 1] == 0)] == 0).all()
    # the goal zone check reports an agent in some steps
    assert 0 < outs["goal"].sum() < outs["goal"].size
    # episodes reset inside the trace: cubes and the ball get new entities
    ent = outs["body_entity"]
    assert not np.array_equal(ent[1], ent[-1])


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_reference_reproduces_golden(name):
    from oracle import runner
    from sims import SIMS
    sim, W, steps, cfg = GOLDENS[name]
    if not runner.available(sim):
        pytest.skip(f"needs oracle/_ref/ref_{sim} (make -C oracle -f overlap.mk overlap)")
    _, _, ins, want = load_golden(name)
    got, _ = runner.run_reference(SIMS[sim], W, steps, ins, cfg, workers=1)
    assert_traces_equal(got, want)


# ---- GPU -----------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_matches_golden(name):
    sim, W, steps, cfg = GOLDENS[name]
    _, _, ins, want = load_golden(name)
    got, n_kernels = rollout_gpu(sim, W, steps, ins, cfg)
    assert n_kernels > 0
    assert sorted(got) == sorted(want)
    assert_traces_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(OVERLAP_REFERENCE_CASES))
def test_matches_reference_digests(case):
    sim, W, steps, ins, cfg = overlap_case(case)
    got, _ = rollout_gpu(sim, W, steps, ins, cfg)
    want = _digests()[case]
    have = trace_digests(got)
    assert sorted(have) == sorted(want)
    assert [k for k in sorted(want) if have[k] != want[k]] == []


@pytest.mark.gpu
def test_triggers_8192_worlds_prefix():
    # Worlds are independent: the first 300 worlds of an 8192-world run step like the
    # 300-world case.  Entity IDs are not comparable across world counts (the singletons
    # take the first W IDs of each kind), so IDs must agree up to a one-to-one relabelling
    # per world and every other value bit for bit.
    case = "triggers_w300_s150"
    _, W, steps, ins, cfg = overlap_case(case)
    small, _ = rollout_gpu("triggers", W, steps, ins, cfg)
    want = _digests()[case]
    have = trace_digests(small)
    assert [k for k in sorted(want) if have[k] != want[k]] == []

    big = 8192
    rest = triggers_inputs(big - W, steps, seed=77)
    ins_big = {k: np.concatenate([v, rest[k]], axis=1) for k, v in ins.items()}
    got, _ = rollout_gpu("triggers", big, steps, ins_big, cfg)
    assert got["agent_pos"][:, :W].view(np.uint32).tolist() == small["agent_pos"].view(np.uint32).tolist()

    cs, ps = _pairs(small)
    cb, pb = _pairs({"pairs": got["pairs"][:, :W]})
    assert np.array_equal(cs, cb)
    assert np.array_equal(ps[..., 2:], pb[..., 2:])
    zs, zb = small["zone"], got["zone"][:, :W]
    other = [c for c in range(zs.shape[-1]) if c != 1]
    assert np.array_equal(zs[..., other], zb[..., other])

    for w in range(W):
        ids_small = np.concatenate([ps[:, w, :, :2].ravel(), zs[:, w, 1]])
        ids_big = np.concatenate([pb[:, w, :, :2].ravel(), zb[:, w, 1]])
        fwd, back = {}, {}
        for a, b in zip(ids_small.tolist(), ids_big.tolist()):
            assert fwd.setdefault(a, b) == b and back.setdefault(b, a) == a, f"world {w}"


@pytest.mark.gpu
@pytest.mark.parametrize("sim,W,steps", [("triggers", 256, 120), ("buttons", 192, 100)])
def test_matches_live_reference(sim, W, steps):
    # a roll-out that no stored trace covers, against the reference binary the build made
    from oracle import runner
    from sims import SIMS
    if not runner.available(sim):
        pytest.skip(f"needs oracle/_ref/ref_{sim} (make -C oracle -f overlap.mk overlap)")
    cfg = {"seed": 4242} if sim == "triggers" else {"episode_len": 45, "seed": 4242}
    ins = INPUTS[sim](W, steps, seed=31)
    want, _ = runner.run_reference(SIMS[sim], W, steps, ins, cfg, workers=4)
    got, _ = rollout_gpu(sim, W, steps, ins, cfg)
    assert sorted(got) == sorted(want)
    assert_traces_equal(got, want)


# ---- GPU: capacity cliffs and misuse --------------------------------------------------------

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
    assert torch.arange(1024, device="cuda").sum().item() == 1023 * 512


@pytest.mark.gpu
def test_candidate_cap_per_world(monkeypatch):
    from sims import make_executor
    monkeypatch.setenv("MADRONA_B200_MAX_CANDIDATES_PER_WORLD", "3")
    ex = make_executor("triggers", 64, seed=3)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 3)
    assert step == 0 and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


# triggers_w300_s150 needs 2133 CandidateTemporary rows in its first step and first needs
# more than 2560 in its 11th (2817 at most); 8 rows / world start the table at 2560
CLIFF_ROWS_PER_WORLD = "8"


@pytest.mark.gpu
def test_candidate_table_overflow_without_growth(monkeypatch):
    from sims import make_executor
    import torch
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", CLIFF_ROWS_PER_WORLD)
    monkeypatch.setenv("MADRONA_B200_TABLE_GROWTH", "0")
    _, W, steps, ins, cfg = overlap_case("triggers_w300_s150")
    ex = make_executor("triggers", W, **cfg)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    act = ex.tensor(0, "int32", (W, 2, 2))
    err_step, msg = None, ""
    import madrona_b200 as mb
    for t in range(steps):
        act.copy_(torch.from_numpy(np.ascontiguousarray(ins["action"][t])))
        try:
            ex.run(graph)
        except mb.MadronaB200Error as e:
            err_step, msg = t, str(e)
            break
    assert err_step == 10 and "table overflow" in msg, (err_step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
def test_candidate_table_grows_between_steps(monkeypatch):
    # the same start size with growth on: the first step's high-water mark (more than half
    # the capacity) doubles the table before the demand passes the start size
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", CLIFF_ROWS_PER_WORLD)
    case = "triggers_w300_s150"
    sim, W, steps, ins, cfg = overlap_case(case)
    got, _ = rollout_gpu(sim, W, steps, ins, cfg)
    have = trace_digests(got)
    want = _digests()[case]
    assert [k for k in sorted(want) if have[k] != want[k]] == []


@pytest.mark.gpu
def test_overlap_tasks_and_solver_in_one_graph_are_rejected():
    import madrona_b200 as mb
    from sims import make_executor
    ex = make_executor("triggers_with_solver", 8, seed=1)
    with pytest.raises(mb.MadronaB200Error, match="setupStandaloneBroadphaseOverlapTasks"):
        ex.buildLaunchGraphAllTaskGraphs()
    _device_still_healthy()
    ex.close()
