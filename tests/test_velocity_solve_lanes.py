"""Both velocity-solve instances against each other and against the reference CPU backend,
around the point where velocitySolveLanes switches: physSolveVelocitiesKernel<16> while the
worlds fit one wave of it (numSMs x 32 worlds, T), physSolveVelocitiesKernel<8> past it (4
worlds per warp sharing n_max / levels_max).

For balls_many (95 bodies), hullpile_many (60 bodies, contacts past the 48 staged ones),
hullpile and crowd at 300 bodies (levels in the global levelScratch rows), each case runs
W = T and W = T + 1 worlds (balls_many also T + 3), all seeded seed + w (pack_init):
- lane check: a torch.profiler trace of one step names the instance each run launches, so a
  change of the rule or of the SM count fails here instead of testing one instance twice;
- cross-lane check: worlds [0, T) are equal between the runs, every frame and every exported
  column but the entity handles (one pool for all worlds);
- tail check: the run's seed is S0 - (T - 4), so worlds [T - 4, W) carry seeds S0, S0 + 1, ...
  whatever the SM count, and must equal worlds 0, 1, ... of a 7-world reference run seeded
  S0.  They hold the last, partly idle warp of both solves (T + 1 is odd).
A world depends on its init seed alone: the sims draw everything from RNG(init.seed), and
entity IDs are handed out in world order at init (the second init pass pre-assigns each
world's 64-ID blocks, state.hpp acquireEntityLocked), so a world's bodies keep their
in-world ID order, which orders its pairs, whatever its index.  The reference traces are
kept as one SHA-256 per world and column (tests/golden/solve_lanes_digests.json, written by
tests/golden/make_solve_lanes_golden.py).  Bit-exact; 1e-4 only with
MADRONA_B200_FAST_MATH=1, against a live reference run."""
import json
import os
import re

import numpy as np
import pytest

from oracle import runner
from sims import SIMS
from trace_utils import GOLDEN_DIR, trace_digests

EXACT = os.environ.get("MADRONA_B200_FAST_MATH", "0") != "1"
DIGESTS_PATH = os.path.join(GOLDEN_DIR, "solve_lanes_digests.json")
S0 = 90000              # seed of the first reference world
TAIL = 4                # worlds below T in the tail check
REF_WORLDS = 7          # T - 4 .. T + 2

MANY_ENV = {"MADRONA_B200_MAX_CANDIDATES_PER_WORLD": "4096", "MADRONA_B200_MAX_CONTACTS_PER_WORLD": "2048",
            "MADRONA_B200_ROWS_PER_WORLD": "128"}
CROWD_BODIES = 300
# scripts/bench_large_physics_worlds.py crowd_env(300)
CROWD_ENV = {"MADRONA_B200_MAX_BODIES_PER_WORLD": "4096", "MADRONA_B200_ROWS_PER_WORLD": str(CROWD_BODIES + 64),
             "MADRONA_B200_PERSIST_BYTES": str(3 << 30),
             "MADRONA_B200_MAX_CANDIDATES_PER_WORLD": str(max(16 * CROWD_BODIES, 1024)),
             "MADRONA_B200_MAX_CONTACTS_PER_WORLD": str(max(8 * CROWD_BODIES, 512))}

# case -> (sim, steps, cfg without the seed, env, world counts past T)
CASES = {
    "balls_many": ("balls_many", 80, {}, MANY_ENV, (1, 3)),
    "hullpile_many": ("hullpile_many", 100, {}, MANY_ENV, (1,)),
    "hullpile": ("hullpile", 100, {}, {}, (1,)),
    "crowd": ("crowd", 60, {"episode_len": 0, "uniform_bodies": CROWD_BODIES}, CROWD_ENV, (1,)),
}


def _compared(sim):
    return [s.name for s in SIMS[sim].outputs if not s.name.endswith("entity")]


def world_traces(sim, frames, first, count):
    """Per world in [first, first + count) of a trace (frames[t][column], numpy, world-major
    rows for the dynamic columns): {column: [steps + 1, ...] array, or a list of per-frame rows
    for a dynamic column}."""
    dynamic = {s.name for s in SIMS[sim].outputs if s.dynamic}
    out = [{} for _ in range(count)]
    for k in _compared(sim):
        for j in range(count):
            out[j][k] = []
    for f in frames:
        offs = None
        if dynamic:
            offs = np.concatenate([[0], np.cumsum(f["body_count"][:, 0])])
        for k in _compared(sim):
            for j in range(count):
                w = first + j
                out[j][k].append(f[k][offs[w]:offs[w + 1]] if k in dynamic else f[k][w])
    for j in range(count):
        for k in _compared(sim):
            if k not in dynamic:
                out[j][k] = np.stack(out[j][k])
    return out


def reference_frames(sim, outs):
    """A reference trace (outputs[name][steps + 1, W, ...] or per-frame row lists) as frames."""
    steps = len(outs["body_pos"]) - 1
    return [{k: v[t] for k, v in outs.items()} for t in range(steps + 1)]


def reference_world_digests(case):
    sim, steps, cfg, _, _ = CASES[case]
    outs, _ = runner.run_reference(SIMS[sim], REF_WORLDS, steps, {}, dict(cfg, seed=S0), workers=1)
    return [trace_digests(w) for w in world_traces(sim, reference_frames(sim, outs), 0, REF_WORLDS)], outs


def _solve_lanes(prof):
    lanes = set()
    for e in prof.events():
        m = re.search(r"physSolveVelocitiesKernel(?:<|ILi)(\d+)", e.name)
        if m and e.device_time_total > 0:
            lanes.add(int(m.group(1)))
    return lanes


def _rollout(sim, W, steps, cfg, visit):
    """Rolls W worlds on the GPU, calls visit(t, frame) with every frame (device tensors,
    entity handles left out); returns the velocity-solve lane counts the first step launched."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from sims import make_executor
    desc = SIMS[sim]
    ex = make_executor(sim, W, **cfg)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    keep = [s for s in desc.outputs if not s.name.endswith("entity")]

    def frame():
        f = {}
        for s in keep:
            if s.dynamic:
                rows = ex.exportedNumRows(s.slot)
                f[s.name] = ex.tensor(s.slot, s.dtype, (max(rows, 1),) + s.per_world)[:rows].clone()
            else:
                f[s.name] = ex.tensor(s.slot, s.dtype, (W,) + s.per_world).clone()
        return f

    visit(0, frame())
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ex.run(graph)
        torch.cuda.synchronize()
    visit(1, frame())
    for t in range(2, steps + 1):
        ex.run(graph)
        visit(t, frame())
    del graph
    ex.close()
    return _solve_lanes(prof)


def _same(a, b):
    import torch
    if a.shape != b.shape:
        return False
    if EXACT or not a.dtype.is_floating_point:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.allclose(a, b, rtol=1e-4, atol=1e-5)


def _prefix(sim, f, T):
    """Worlds [0, T) of a device frame."""
    dynamic = {s.name for s in SIMS[sim].outputs if s.dynamic}
    rows = int(f["body_count"][:T, 0].sum().item()) if dynamic else None
    return {k: (v[:rows] if k in dynamic else v[:T]) for k, v in f.items()}


def _check_tail(case, sim, tail, first_ref):
    """tail: per-world traces of worlds [T - 4, W) of a GPU run; they carry the seeds of
    reference worlds first_ref, first_ref + 1, ..."""
    if EXACT:
        with open(DIGESTS_PATH) as f:
            want = json.load(f)[case]
        for j, w in enumerate(tail):
            have = trace_digests(w)
            assert sorted(have) == sorted(want[first_ref + j])
            differ = [k for k in sorted(have) if have[k] != want[first_ref + j][k]]
            assert not differ, f"{case}: world T - {TAIL - j} differs from the reference in {differ}"
        return
    if not runner.available(sim):
        pytest.skip("a tolerance comparison needs the reference CPU backend (oracle/_ref)")
    _, outs = reference_world_digests(case)
    ref = world_traces(sim, reference_frames(sim, outs), 0, REF_WORLDS)
    for j, w in enumerate(tail):
        for k, v in w.items():
            for g, r in zip(v if isinstance(v, list) else [v], ref[first_ref + j][k] if isinstance(v, list)
                            else [ref[first_ref + j][k]]):
                assert g.shape == r.shape, (case, k)
                np.testing.assert_allclose(g, r, rtol=1e-4, atol=1e-5, err_msg=f"{case} {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_velocity_solve_lanes_match_each_other_and_the_reference(monkeypatch, case):
    import torch
    sim, steps, cfg, env, extra = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    T = torch.cuda.get_device_properties(0).multi_processor_count * 32
    cfg = dict(cfg, seed=S0 - (T - TAIL))
    assert cfg["seed"] >= 0

    def to_host(f, first, last):
        dynamic = {s.name for s in SIMS[sim].outputs if s.dynamic}
        out = {}
        if dynamic:
            counts = f["body_count"][:, 0].cpu().numpy()
            offs = np.concatenate([[0], np.cumsum(counts)])
            out["body_count"] = np.ascontiguousarray(f["body_count"][first:last].cpu().numpy())
            for k in dynamic:
                if k in f:
                    out[k] = f[k][offs[first]:offs[last]].cpu().numpy()
        else:
            out = {k: v[first:last].cpu().numpy() for k, v in f.items()}
        return out

    # 16 lanes: keep worlds [0, T) of every frame on the device
    wide, wide_tail = [], []

    def keep(t, f):
        wide.append(f)
        wide_tail.append(to_host(f, T - TAIL, T))

    lanes = _rollout(sim, T, steps, cfg, keep)
    assert lanes == {16}, f"{T} worlds launched physSolveVelocitiesKernel{sorted(lanes)}, want <16>"
    _check_tail(case, sim, world_traces(sim, wide_tail, 0, TAIL), 0)

    for more in extra:
        W = T + more
        narrow_tail, differ = [], []

        def compare(t, f):
            got = _prefix(sim, f, T)
            for k, v in wide[t].items():
                if not _same(got[k], v):
                    differ.append((t, k))
            narrow_tail.append(to_host(f, T - TAIL, W))

        lanes = _rollout(sim, W, steps, cfg, compare)
        assert lanes == {8}, f"{W} worlds launched physSolveVelocitiesKernel{sorted(lanes)}, want <8>"
        assert not differ, f"{case}: worlds [0, {T}) differ between 16 and 8 lanes at (step, column) {differ[:5]}"
        _check_tail(case, sim, world_traces(sim, narrow_tail, 0, TAIL + more), 0)
