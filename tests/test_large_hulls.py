"""Convex hulls past the narrowphase's staging caps (16 vertices, 16 faces, 8-vertex faces),
accepted with MADRONA_B200_MAX_HULL_SIZE: the hullpile simulators with 24-gon prisms, a
16-gon bipyramid, an icosphere and an 11-gon pyramid (sims/objects.py hullpile_big_specs), GPU
engine vs the reference CPU backend.  Same bar as tests/test_hullpile.py: every exported
column BIT-EXACT (1e-4 only with MADRONA_B200_FAST_MATH=1).  The pairs with such a hull run
in physNarrowphaseLargeKernel (one warp per pair), the others in the same step on the
group-per-pair path.  What the goldens exercise is checked by tests/test_large_hull_model.py.
Only Solver::XPBD: the hullpile simulators have no TGS build (the reference's TGS makes no
contacts, so it has no narrowphase result to compare)."""
import dataclasses
import json
import os
from functools import partial

import numpy as np
import pytest

from oracle import runner
from sims import SIMS
from trace_utils import GOLDEN_DIR, assert_traces_equal, load_golden, rollout_gpu, trace_digests

EXACT = os.environ.get("MADRONA_B200_FAST_MATH", "0") != "1"
KNOB = "MADRONA_B200_MAX_HULL_SIZE"
# the icosphere has 80 faces
FITS_ALL = "96"
MANY_ENV = {"MADRONA_B200_MAX_CANDIDATES_PER_WORLD": "4096", "MADRONA_B200_MAX_CONTACTS_PER_WORLD": "2048",
            "MADRONA_B200_ROWS_PER_WORLD": "128"}

# golden name -> (sim, worlds, steps, cfg); written by tests/golden/make_large_hull_golden.py
GOLDENS = {
    "hullpile_big_w4_s150": ("hullpile_big", 4, 150, {"seed": 41}),
    "hullpile_big_many_w2_s100": ("hullpile_big_many", 2, 100, {"seed": 50}),
}
# Roll-outs kept as one SHA-256 per column of the reference CPU backend's trace (the scheme of
# trace_utils.REFERENCE_CASES, in a file of their own): name -> (sim, worlds, steps, cfg)
LARGE_REFERENCE_CASES = {
    "hullpile_big_w128_s100": ("hullpile_big", 128, 100, {"seed": 62000}),
    "hullpile_big_w64_s60": ("hullpile_big", 64, 60, {"seed": 64000}),
}
LARGE_DIGESTS_PATH = os.path.join(GOLDEN_DIR, "large_hull_digests.json")


def reference_desc(sim):
    """The descriptor to hand to oracle.runner for `sim`: the large-hull fixtures are the
    hullpile simulators with other objects, so they run on the hullpile reference binaries
    (which always build the pile layout)."""
    name = {"hullpile_big": "hullpile", "hullpile_big_many": "hullpile_many"}[sim]
    return dataclasses.replace(SIMS[sim], name=name)


def _assert_matches_digests(case, got, skip=()):
    sim, W, steps, cfg = LARGE_REFERENCE_CASES[case]
    if not EXACT:
        if not runner.available(reference_desc(sim).name):
            pytest.skip("a tolerance comparison needs the reference CPU backend (oracle/_ref)")
        ref, _ = runner.run_reference(reference_desc(sim), W, steps, {}, cfg, workers=4)
        assert_traces_equal({k: v for k, v in got.items() if k not in skip},
                            {k: v for k, v in ref.items() if k not in skip}, exact=False, rtol=1e-4, atol=1e-5)
        return
    with open(LARGE_DIGESTS_PATH) as f:
        want = json.load(f)[case]
    have = trace_digests(got)
    differ = [k for k in sorted(want) if k not in skip and have.get(k) != want[k]]
    assert not differ, f"{case}: columns differ from the reference CPU backend: {differ}"


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


# ---- the goldens themselves (no GPU) ------------------------------------------------------------

@pytest.mark.parametrize("golden", sorted(GOLDENS))
def test_golden_is_finite_and_above_the_floor(golden):
    W, steps, ins, outs = load_golden(golden)
    for k in ("body_pos", "body_rot", "body_vel"):
        assert np.isfinite(outs[k]).all(), k
    pos = outs["body_pos"]
    # body 0 is the plane; every other body keeps its centre above it and inside the pen
    assert pos[:, :, 1:, 2].min() > 0.05
    assert np.abs(pos[:, :, :, :2]).max() <= 6.25


@pytest.mark.skipif(not runner.available("hullpile_many"), reason="oracle/_ref not built")
@pytest.mark.parametrize("golden", sorted(GOLDENS))
def test_reference_backend_reproduces_golden(golden):
    sim, W, steps, cfg = GOLDENS[golden]
    _, _, ins, outs = load_golden(golden)
    got, _ = runner.run_reference(reference_desc(sim), W, steps, ins, cfg, workers=1)
    assert_traces_equal(got, outs)


# ---- GPU ------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("max_hull_size", [FITS_ALL, "255"])
def test_gpu_matches_golden(monkeypatch, max_hull_size):
    # two sizes of the per-warp stage in shared memory, the same bits
    monkeypatch.setenv(KNOB, max_hull_size)
    sim, W, steps, cfg = GOLDENS["hullpile_big_w4_s150"]
    _, _, ins, outs = load_golden("hullpile_big_w4_s150")
    got, n_kernels = rollout_gpu(sim, W, steps, ins, cfg)
    assert n_kernels > 10
    assert_traces_equal(got, outs, exact=EXACT, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_many_gpu_matches_golden(monkeypatch):
    for k, v in MANY_ENV.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv(KNOB, FITS_ALL)
    sim, W, steps, cfg = GOLDENS["hullpile_big_many_w2_s100"]
    _, _, ins, outs = load_golden("hullpile_big_many_w2_s100")
    assert outs["body_pos"].shape[2] == 60
    got, _ = rollout_gpu(sim, W, steps, ins, cfg)
    assert_traces_equal(got, outs, exact=EXACT, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_gpu_matches_live_reference_many_worlds(monkeypatch):
    monkeypatch.setenv(KNOB, FITS_ALL)
    sim, W, steps, cfg = LARGE_REFERENCE_CASES["hullpile_big_w128_s100"]
    got, _ = rollout_gpu(sim, W, steps, {}, cfg)
    _assert_matches_digests("hullpile_big_w128_s100", got)


@pytest.mark.gpu
def test_4096_worlds_prefix_equals_reference(monkeypatch):
    # worlds are independent and seeded by their index: worlds [0, 64) of a 4096-world run
    # (the large kernel's persistent grid full of pairs) equal a 64-world reference run
    from test_full_size import _rollout_prefix
    monkeypatch.setenv(KNOB, FITS_ALL)
    sim, keep, steps, cfg = LARGE_REFERENCE_CASES["hullpile_big_w64_s60"]
    got = _rollout_prefix(sim, 4096, steps, {}, cfg, keep)
    # handles come from one pool for all worlds
    _assert_matches_digests("hullpile_big_w64_s60", got, skip=("body_entity",))


@pytest.mark.gpu
def test_24_gon_face_on_face_and_on_the_plane(monkeypatch):
    # the 24-gon prism face down on the static 24-gon pedestal at a relative yaw (a 24-gon
    # clipped against a 24-gon: up to 48 points before the reduction) and on the plane (a
    # 24-point incident face): no error, and it rests where the octagonal prism of
    # tests/test_cliffs.py rests
    from sims import make_executor
    monkeypatch.setenv(KNOB, "64")
    for layout in (1, 2):
        ex = make_executor("hullpile_big", 8, layout=layout, seed=1)
        graph = ex.buildLaunchGraphAllTaskGraphs()
        step, msg = _run_until_error(ex, graph, 10)
        assert step is None, (layout, step, msg)
        rows = ex.exportedNumRows(0)
        assert rows == 8 * (3 if layout == 1 else 2)
        pos = ex.tensor(0, "float32", (rows, 3)).cpu().numpy().reshape(8, -1, 3)
        assert np.allclose(pos[:, -1, 2], 2.0 if layout == 1 else 0.5, atol=0.05), pos[:, -1]
        ex.close()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", [1, 2], ids=["hull_on_hull", "hull_on_plane"])
def test_11_gon_pyramids_run_with_the_knob(monkeypatch, layout):
    # the two layouts that raise without the knob (tests/test_cliffs.py
    # test_hull_face_vertex_cap): 12 vertices and 12 faces, large only through the base.
    # Base to base at a relative yaw of pi / 11 (a clip to 22 points), or base down on the plane
    from sims import make_executor
    from sims.objects import hullpile_objects
    monkeypatch.setenv(KNOB, "32")
    ex = make_executor("hullpile", 8, objects_fn=partial(hullpile_objects, big_face=True), layout=layout, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 10)
    assert step is None, (step, msg)
    rows = ex.exportedNumRows(0)
    pos = ex.tensor(0, "float32", (rows, 3)).cpu().numpy().reshape(8, -1, 3)
    assert np.allclose(pos[:, -1, 2], 2.0 if layout == 1 else 0.5, atol=0.05), pos[:, -1]
    ex.close()


@pytest.mark.gpu
@pytest.mark.parametrize("sim,golden,cfg", [("hullpile", "hullpile_w4_s150", {"seed": 41}),
                                            ("room", "room_w4_s210", {"episode_len": 100, "seed": 21})])
def test_small_hull_fixtures_are_unchanged_by_the_knob(monkeypatch, sim, golden, cfg):
    # no primitive is large: the same trace from the same number of kernels
    W, steps, ins, outs = load_golden(golden)
    _, plain_kernels = rollout_gpu(sim, W, 1, {k: v[:1] for k, v in ins.items()} or None, cfg)
    monkeypatch.setenv(KNOB, "255")
    got, n_kernels = rollout_gpu(sim, W, steps, ins or None, cfg)
    assert n_kernels == plain_kernels
    assert_traces_equal(got, outs, exact=EXACT, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_large_hulls_add_one_kernel_per_substep(monkeypatch):
    from sims import make_executor
    counts = {}
    for size in (None, FITS_ALL):
        if size:
            monkeypatch.setenv(KNOB, size)
        ex = make_executor("hullpile_big", 4, seed=41)
        graph = ex.buildLaunchGraphAllTaskGraphs()
        counts[size] = graph.num_kernels
        del graph
        ex.close()
    assert counts[FITS_ALL] == counts[None] + 4     # sims/hullpile runs 4 substeps


@pytest.mark.gpu
def test_hull_past_the_knob_raises(monkeypatch):
    # the 42-vertex, 80-face icosphere with room for 32: flagged by the pair's first test
    from sims import make_executor
    monkeypatch.setenv(KNOB, "32")
    ex = make_executor("hullpile_big", 8, seed=41)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 120)
    assert step is not None and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
def test_large_hull_without_the_knob_raises_at_step_0():
    # default: the 24-gon prism already touches its pedestal's box at step 0
    from sims import make_executor
    ex = make_executor("hullpile_big", 8, layout=1, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    step, msg = _run_until_error(ex, graph, 2)
    assert step == 0 and "physics buffer overflow" in msg, (step, msg)
    _device_still_healthy()
    ex.close()


@pytest.mark.gpu
@pytest.mark.parametrize("value", ["8", "256", "abc", "64x"])
def test_bad_knob_value_fails_executor_creation(monkeypatch, value):
    import madrona_b200 as mb
    from sims import make_executor
    monkeypatch.setenv(KNOB, value)
    with pytest.raises(mb.MadronaB200Error, match=KNOB):
        make_executor("hullpile", 4, seed=1)
    _device_still_healthy()


@pytest.mark.gpu
def test_snapshot_restore_with_large_hulls(monkeypatch):
    # the third pair list is per-step scratch and the class table is immutable: neither is
    # part of a snapshot, and "save, step, restore, step" repeats bit for bit
    from sims import make_executor
    monkeypatch.setenv(KNOB, FITS_ALL)
    W = 16
    ex = make_executor("hullpile_big", W, seed=41)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    cols = [(0, (W, 20, 3)), (1, (W, 20, 4)), (2, (W, 20, 6))]

    def read():
        return [ex.tensor(slot, "float32", shape).cpu().numpy().copy() for slot, shape in cols]

    for _ in range(40):
        ex.run(graph)
    with ex.snapshot() as snap:
        snap.save()
        for _ in range(20):
            ex.run(graph)
        first = read()
        snap.restore()
        for _ in range(20):
            ex.run(graph)
        second = read()
    for a, b in zip(first, second):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert not np.array_equal(first[0], np.zeros_like(first[0]))
    ex.close()
