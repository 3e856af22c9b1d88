"""Capacity cliffs (DESIGN.md 3.4): every documented limit must FAIL LOUDLY -- run()
raises with the matching message -- and leave the executor usable enough to be
queried and destroyed (no sticky illegal-address error, no out-of-bounds write:
the next CUDA call still succeeds)."""
import numpy as np
import pytest

from trace_utils import make_inputs


def _run_until_error(ex, graph, steps, inputs=None, in_tensors=None):
    import torch
    import madrona_b200 as mb
    for t in range(steps):
        if inputs is not None:
            for k, tens in in_tensors.items():
                tens.copy_(torch.from_numpy(np.ascontiguousarray(inputs[k][t])))
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


@pytest.mark.gpu
def test_dynamic_table_overflow_is_reported_at_the_reset_step(monkeypatch):
    # room: 31 rows / world at rest, 46 while a reset has destroyed-but-uncompacted cubes
    from sims import make_executor
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "36")
    monkeypatch.setenv("MADRONA_B200_TABLE_GROWTH", "0")     # growth off: the raw capacity cliff
    W = 64
    ex = make_executor("room", W, episode_len=6, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 12)
    assert step == 5 and "table overflow" in msg, (step, msg)
    # the error is sticky, the row count stayed inside the allocation
    assert ex.exportedNumRows(9) <= 36 * W + 255
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
def test_table_overflow_during_world_construction(monkeypatch):
    import madrona_b200 as mb
    from sims import make_executor
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "4")
    monkeypatch.setenv("MADRONA_B200_TABLE_GROWTH", "0")
    with pytest.raises(mb.MadronaB200Error, match="table overflow"):
        make_executor("gridworld", 512, grid_size=6, episode_len=20, init_items=20, seed=0)
    _device_still_healthy()


@pytest.mark.gpu
@pytest.mark.parametrize("var,value", [("MADRONA_B200_MAX_CANDIDATES_PER_WORLD", "8"),
                                       ("MADRONA_B200_MAX_CONTACTS_PER_WORLD", "4")])
def test_candidate_and_contact_caps(monkeypatch, var, value):
    from sims import make_executor
    monkeypatch.setenv(var, value)
    ex = make_executor("room", 32, episode_len=50, seed=3)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 3)
    assert step == 0 and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
def test_body_cap_per_world(monkeypatch):
    # 145 bodies per world: past the candidate search's per-world body cap
    from sims import make_executor
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "160")
    ex = make_executor("balls_cliff", 4, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 2)
    assert step == 0 and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
def test_hull_vertex_cap():
    # cubes replaced by 20-vertex prisms: hull - hull / hull - plane pairs beyond the
    # 16-vertex staging cap must raise, not overrun the staging arrays
    from sims import make_executor
    from sims.objects import room_objects_big_hull
    W = 16
    ex = make_executor("room", W, objects_fn=room_objects_big_hull, episode_len=50, seed=2)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    ins = make_inputs("room", W, 40, seed=3)
    act = ex.tensor(1, "int32", (W, 2, 3))
    step, msg = _run_until_error(ex, graph, 40, {"action": ins["action"]}, {"action": act})
    assert step is not None and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [1, 2], ids=["hull_on_hull", "hull_on_plane"])
def test_hull_face_vertex_cap(layout):
    # 11-gon pyramids: 12 vertices and 12 faces, inside the hull caps, but an 11-vertex
    # base.  Base to base on an upside-down static one at a relative yaw of pi / 11 (a
    # hull - hull pair whose clip would make 22 points: tests/test_hull_clip_model.py), or
    # base down on the plane (the incident face of a hull - plane pair): both must raise
    # at step 0, not overrun the 8-vertex face staging or the 20-point clip buffers
    from functools import partial
    from sims import make_executor
    from sims.objects import hullpile_objects
    ex = make_executor("hullpile", 8, objects_fn=partial(hullpile_objects, big_face=True), layout=layout, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 2)
    assert step == 0 and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
def test_hull_face_on_face_at_the_cap_runs():
    # the same two layouts with the octagonal prism: 8-vertex faces are within the cap
    from sims import make_executor
    for layout in (1, 2):
        ex = make_executor("hullpile", 8, layout=layout, seed=1)
        graph = ex.buildLaunchGraphAllTaskGraphs()
        step, msg = _run_until_error(ex, graph, 10)
        assert step is None, (layout, step, msg)
        rows = ex.exportedNumRows(0)
        assert rows == 8 * (3 if layout == 1 else 2)
        pos = ex.tensor(0, "float32", (rows, 3)).cpu().numpy().reshape(8, -1, 3)
        # the prism (each world's last body) rests on the pedestal's face (z = 1.5) or on
        # the plane, its centre 0.5 above
        assert np.allclose(pos[:, -1, 2], 2.0 if layout == 1 else 0.5, atol=0.05), pos[:, -1]
        ex.close()


# ---- table growth (role of the reference's VM-backed tables, src/mw/device/state.cpp:29-80) ----

@pytest.mark.gpu
def test_tables_grow_during_world_construction(monkeypatch):
    # 4 rows / world of initial capacity, 20 items / world to create: construction must
    # double the table until the worlds fit, and the run must equal the golden trace
    from trace_utils import assert_traces_equal, load_golden, rollout_gpu
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "4")
    W, steps, ins, outs = load_golden("gridworld_w5_s400")
    got, _ = rollout_gpu("gridworld", W, 150, {k: v[:150] for k, v in ins.items()},
                         {"grid_size": 3, "episode_len": 97, "init_items": 20, "seed": 3})
    assert_traces_equal(got, {k: v[:151] for k, v in outs.items()})


@pytest.mark.gpu
def test_tables_grow_between_steps(monkeypatch):
    # room: 31 body rows / world at rest, 46 while a reset waits for compaction; with 36
    # rows / world to start with, the table must have been grown (between steps, from the
    # high-water mark) before the reset at step 100 -- results unchanged, exported pointers stable
    from sims import make_executor
    from trace_utils import load_golden
    import torch
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "36")
    W, steps, ins, outs = load_golden("room_w4_s210")
    ex = make_executor("room", W, episode_len=100, seed=21)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    ptr_before = ex.getExported(9)
    act, reset = ex.tensor(1, "int32", (W, 2, 3)), ex.tensor(0, "int32", (W, 1))
    for t in range(120):
        act.copy_(torch.from_numpy(np.ascontiguousarray(ins["action"][t])))
        reset.copy_(torch.from_numpy(np.ascontiguousarray(ins["reset"][t])))
        ex.run(graph)
        rows = ex.exportedNumRows(9)
        pos = ex.tensor(9, "float32", (rows, 3)).cpu().numpy()
        assert np.array_equal(pos.view(np.uint32), outs["body_pos"][t + 1].view(np.uint32)), t
    assert ex.getExported(9) == ptr_before
    ex.close()
