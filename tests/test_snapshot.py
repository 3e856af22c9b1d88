"""Executor snapshots (include/madrona_b200.h mb2_snapshot_*, kernels_snapshot.cu): the engine
is deterministic step to step, so "save, step, restore, step" must reproduce every exported
column bit for bit, and where a golden trace of the reference CPU backend exists both passes
after the save must still match it."""
import os
import subprocess

import numpy as np
import pytest

import madrona_b200 as mb
from sims import SIMS, make_executor
from sims.inputs import buttons_inputs, triggers_inputs
from trace_utils import assert_traces_equal, load_golden, make_inputs

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(sim, W, steps, seed=1):
    if sim == "triggers":
        return triggers_inputs(W, steps, seed=seed)
    if sim == "buttons":
        return buttons_inputs(W, steps, seed=seed)
    if sim in ("room_render",):
        return make_inputs("room", W, steps, seed=seed)
    if not SIMS[sim].inputs:
        return {}
    return make_inputs(sim, W, steps, seed=seed)


class Driver:
    """A fixture executor stepped with recorded inputs; columns() is the raw bytes and row
    count of every exported column."""

    def __init__(self, sim, W, ins, **cfg):
        self.desc = SIMS[sim]
        self.W = W
        self.ex = make_executor(sim, W, **cfg)
        self.graph = self.ex.buildLaunchGraphAllTaskGraphs()
        self.render = self.ex.buildRenderGraph() if self.desc.render is not None else None
        self.ins = ins
        self.in_t = {s.name: self.ex.tensor(s.slot, s.dtype, (W,) + s.per_world) for s in self.desc.inputs}

    def step(self, t):
        import torch
        for name, arr in self.ins.items():
            self.in_t[name].copy_(torch.from_numpy(np.ascontiguousarray(arr[t])))
        torch.cuda.synchronize()
        self.ex.run(self.graph)

    def columns(self):
        out = {}
        for slot in range(self.desc.num_exports):
            try:
                self.ex.getExported(slot)
            except mb.MadronaB200Error:
                continue
            rows, rb = self.ex.exportedNumRows(slot), self.ex.exportedRowBytes(slot)
            n = rows * rb
            data = self.ex.tensor(slot, "uint8", (max(n, 1),))[:n].cpu().numpy().copy()
            out[slot] = (rows, data)
        return out

    def outputs(self):
        """The fixture's named outputs in the layout of tests/trace_utils.rollout_gpu."""
        frame = {}
        for s in self.desc.outputs:
            if s.dynamic:
                rows = self.ex.exportedNumRows(s.slot)
                t = self.ex.tensor(s.slot, s.dtype, (max(rows, 1),) + s.per_world)
                frame[s.name] = t.cpu().numpy()[:rows].copy()
            else:
                frame[s.name] = self.ex.tensor(s.slot, s.dtype, (self.W,) + s.per_world).cpu().numpy().copy()
        return frame

    def close(self):
        self.graph = self.render = None
        self.ex.close()


def _assert_same_columns(a, b, what):
    assert sorted(a) == sorted(b), what
    for slot in a:
        assert a[slot][0] == b[slot][0], f"{what}: export slot {slot} has {b[slot][0]} rows, not {a[slot][0]}"
        assert np.array_equal(a[slot][1], b[slot][1]), f"{what}: export slot {slot} differs"


def _replay(d, steps, record):
    frames = [record()]
    for t in steps:
        d.step(t)
        frames.append(record())
    return frames


# sim -> (worlds, cfg): short episodes, so that resets (entity destruction, creation and
# compaction) fall between the save and the end of the round trip
ROUND_TRIP = {
    "cartpole": (8, {"max_steps": 9}),
    "gridworld": (32, {"grid_size": 6, "episode_len": 10, "init_items": 6, "seed": 11}),
    "room": (4, {"episode_len": 12, "seed": 21}),
    "room_tgs": (3, {"episode_len": 12, "seed": 300}),
    "balls": (6, {"seed": 3}),
    "arena": (2, {"episode_len": 12, "seed": 17}),
    "triggers": (3, {"seed": 11}),
    "buttons": (4, {"episode_len": 12, "seed": 21}),
    "navmesh": (9, {"episode_len": 10, "seed": 5}),
    "customnodes": (23, {"seed": 7}),
}
K, M = 7, 16


@pytest.mark.parametrize("sim", sorted(ROUND_TRIP))
def test_round_trip_is_bit_identical(sim):
    W, cfg = ROUND_TRIP[sim]
    d = Driver(sim, W, _inputs(sim, W, K + M), **cfg)
    for t in range(K):
        d.step(t)
    with d.ex.snapshot() as snap:
        assert snap.nbytes > 0 and snap.saved_nbytes == 0
        snap.save()
        assert 0 < snap.saved_nbytes <= snap.nbytes
        first = _replay(d, range(K, K + M), d.columns)
        snap.restore()
        second = _replay(d, range(K, K + M), d.columns)
    for i, (a, b) in enumerate(zip(first, second)):
        _assert_same_columns(a, b, f"{sim} step {K + i}")
    # the round trip crossed state changes: something moved after the save
    assert any(not np.array_equal(first[0][s][1], first[-1][s][1]) for s in first[0])
    d.close()


GOLDEN_CASES = {
    "gridworld_w32_s150": ("gridworld", {"grid_size": 6, "episode_len": 40, "init_items": 6, "seed": 11}),
    "arena_w2_s200": ("arena", {"episode_len": 90, "seed": 17}),
    "room_w4_s210": ("room", {"episode_len": 100, "seed": 21}),
}


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_both_passes_after_a_mid_trace_save_match_the_reference(name):
    sim, cfg = GOLDEN_CASES[name]
    W, steps, ins, outs = load_golden(name)
    k = steps // 3
    d = Driver(sim, W, ins, **cfg)
    for t in range(k):
        d.step(t)
    want = {n: v[k:] for n, v in outs.items()}
    with d.ex.snapshot() as snap:
        snap.save()
        for attempt in range(2):
            if attempt:
                snap.restore()
            frames = _replay(d, range(k, steps), d.outputs)
            got = {n: [f[n] for f in frames] for n in frames[0]}
            dyn = {s.name for s in d.desc.outputs if s.dynamic}
            got = {n: (v if n in dyn else np.stack(v)) for n, v in got.items()}
            assert_traces_equal(got, want)
    d.close()


@pytest.mark.parametrize("sim,cfg", [
    ("gallery", {"num_props": 40, "resolution": 32, "seed": 5}),
    ("gallery_sized", {"props": [30, 70], "layouts": [0, 1], "width": 48, "height": 20, "seed": 5}),
    ("room_render", {"episode_len": 12, "seed": 3, "resolution": 32, "rgbd": True}),
])
def test_render_after_restore_matches_render_at_save(sim, cfg):
    W = 2 if sim.startswith("gallery") else 4
    d = Driver(sim, W, _inputs(sim, W, 12), **cfg)
    for t in range(3):
        d.step(t)
    d.ex.run(d.render)
    at_save = d.columns()
    with d.ex.snapshot() as snap:
        snap.save()
        for t in range(3, 8):
            d.step(t)
            d.ex.run(d.render)
        assert any(not np.array_equal(at_save[s][1], v[1]) for s, v in d.columns().items())
        snap.restore()
        _assert_same_columns(at_save, d.columns(), f"{sim} after restore")
        d.ex.run(d.render)
        _assert_same_columns(at_save, d.columns(), f"{sim} rendered after restore")
    d.close()


def test_restore_after_the_tables_grew(monkeypatch):
    # room: 31 body rows per world at rest, 46 while a reset waits for compaction; with 36 rows
    # per world to start with the body table grows at the first reset -- after the save
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "36")
    W, steps = 4, 40
    d = Driver("room", W, _inputs("room", W, steps, seed=4), episode_len=20, seed=21)
    for t in range(3):
        d.step(t)
    with d.ex.snapshot() as snap:
        snap.save()
        small = snap.nbytes
        first = _replay(d, range(3, steps), d.columns)
        with d.ex.snapshot() as later:
            assert later.nbytes > small, "the tables did not grow after the save"
        snap.restore()
        assert snap.nbytes == small
        second = _replay(d, range(3, steps), d.columns)
    for i, (a, b) in enumerate(zip(first, second)):
        _assert_same_columns(a, b, f"step {3 + i}")
    d.close()


def test_a_save_after_growth_enlarges_the_snapshot(monkeypatch):
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "36")
    W, steps = 4, 50
    d = Driver("room", W, _inputs("room", W, steps, seed=6), episode_len=20, seed=21)
    with d.ex.snapshot() as snap:
        snap.save()
        small = snap.nbytes
        for t in range(30):
            d.step(t)
        snap.save()
        assert snap.nbytes > small, "the tables did not grow, or the save did not enlarge the snapshot"
        first = _replay(d, range(30, steps), d.columns)
        snap.restore()
        second = _replay(d, range(30, steps), d.columns)
    for i, (a, b) in enumerate(zip(first, second)):
        _assert_same_columns(a, b, f"step {30 + i}")
    d.close()


def test_branches_on_a_torch_stream_equal_straight_runs():
    """Save A, step, save B, restore A, step other inputs, restore B, step: all on one torch
    stream with runAsync, the host never waiting in between."""
    import torch
    W, k, m = 4, 6, 10
    cfg = {"episode_len": 9, "seed": 21}
    main = make_inputs("room", W, k + 2 * m, seed=8)
    other = make_inputs("room", W, k + 2 * m, seed=9)
    alt = {n: np.concatenate([main[n][:k], other[n][k:]]) for n in main}
    fixed = [s for s in SIMS["room"].outputs if not s.dynamic]

    def straight(ins, n):
        d = Driver("room", W, ins, **cfg)
        for t in range(n):
            d.step(t)
        out = {s.name: d.ex.tensor(s.slot, s.dtype, (W,) + s.per_world).cpu().numpy().copy() for s in fixed}
        d.close()
        return out

    d = Driver("room", W, {}, **cfg)
    dev = {n: torch.from_numpy(main[n]).cuda() for n in main}
    dev_alt = {n: torch.from_numpy(alt[n]).cuda() for n in alt}
    outs = {s.name: d.ex.tensor(s.slot, s.dtype, (W,) + s.per_world) for s in fixed}
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    results = {}
    with d.ex.snapshot() as a, d.ex.snapshot() as b:
        with torch.cuda.stream(stream):
            def run(src, steps):
                for t in steps:
                    for n, v in src.items():
                        d.in_t[n].copy_(v[t])
                    d.ex.runAsync(d.graph, stream)

            run(dev, range(k))
            a.save(stream)
            run(dev, range(k, k + m))
            b.save(stream)
            a.restore(stream)
            run(dev_alt, range(k, k + m))
            results["alt"] = {n: t.clone() for n, t in outs.items()}
            b.restore(stream)
            run(dev, range(k + m, k + 2 * m))
            results["main"] = {n: t.clone() for n, t in outs.items()}
        stream.synchronize()
    want = {"main": straight(main, k + 2 * m), "alt": straight(alt, k + m)}
    for branch in ("main", "alt"):
        for n, v in results[branch].items():
            assert np.array_equal(v.cpu().numpy(), want[branch][n]), f"branch {branch}: {n} differs"
    d.close()


def test_misuse_is_rejected_with_a_message():
    lib = mb.load_library()
    d1 = Driver("cartpole", 8, {})
    d2 = Driver("cartpole", 8, {})
    for _ in range(3):
        d1.step(0)
    before = d1.columns()
    snap = d1.ex.snapshot()
    with pytest.raises(mb.MadronaB200Error, match="never saved"):
        snap.restore()
    snap.save()
    assert lib.mb2_snapshot_restore(d2.ex._h, snap._h, None) == 1
    assert b"another executor" in lib.mb2_last_error()
    assert lib.mb2_snapshot_save(d2.ex._h, snap._h, None) == 1
    assert b"another executor" in lib.mb2_last_error()
    assert lib.mb2_snapshot_save(None, snap._h, None) == 1
    assert b"null" in lib.mb2_last_error()
    assert lib.mb2_snapshot_restore(d1.ex._h, None, None) == 1
    assert b"null" in lib.mb2_last_error()
    assert lib.mb2_snapshot_create(None) is None
    assert b"null" in lib.mb2_last_error()
    assert lib.mb2_snapshot_bytes(None) == -1
    _assert_same_columns(before, d1.columns(), "after rejected calls")
    snap.close()
    with pytest.raises(mb.MadronaB200Error, match="closed"):
        snap.save()
    d1.close()
    d2.close()


def test_closing_the_executor_closes_its_snapshots():
    d = Driver("cartpole", 4, {})
    snap = d.ex.snapshot()
    snap.save()
    d.close()
    assert snap.nbytes == 0
    snap.close()


def test_facade_snapshot_round_trip(tmp_path):
    exe = str(tmp_path / "facade_snapshot")
    cmd = ["g++", "-std=c++20", "-O1", "-I" + os.path.join(ROOT, "madrona_b200", "host"),
           os.path.join(ROOT, "tests", "cpp", "facade_snapshot.cpp"), "-o", exe,
           "-L" + os.path.join(ROOT, "madrona_b200"), "-lmadrona_b200",
           "-Wl,-rpath," + os.path.join(ROOT, "madrona_b200"),
           "-L/usr/local/cuda/lib64", "-lcudart"]
    subprocess.run(cmd, check=True, capture_output=True)
    res = subprocess.run([exe, os.path.join(ROOT, "sims", "cartpole", "sim.cpp")],
                         capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    assert "snapshot ok" in res.stdout
