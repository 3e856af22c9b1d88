"""Shared helpers for parity tests: seeded synthetic inputs, GPU roll-outs
through the C ABI, golden fixture I/O."""
from __future__ import annotations

import hashlib
import json
import os
from typing import Dict

import numpy as np

from sims import SIMS, make_executor

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def make_inputs(sim: str, num_worlds: int, num_steps: int, seed: int = 0) -> Dict[str, np.ndarray]:
    rng = np.random.default_rng(seed)
    if sim == "cartpole":
        return {
            "reset": (rng.random((num_steps, num_worlds, 1)) < 0.01).astype(np.int32),
            "action": rng.integers(0, 2, size=(num_steps, num_worlds, 1), dtype=np.int32),
        }
    if sim == "gridworld":
        return {
            "reset": (rng.random((num_steps, num_worlds, 1)) < 0.02).astype(np.int32),
            "action": rng.integers(0, 5, size=(num_steps, num_worlds, 2), dtype=np.int32),
        }
    if sim in ("room", "room_tgs"):
        # mostly "full speed ahead" so agents reach cubes, walls and each other
        amount = np.where(rng.random((num_steps, num_worlds, 2)) < 0.7, 3,
                          rng.integers(0, 4, size=(num_steps, num_worlds, 2)))
        angle = np.where(rng.random((num_steps, num_worlds, 2)) < 0.7, 0,
                         rng.integers(0, 8, size=(num_steps, num_worlds, 2)))
        act = np.stack([amount, angle,
                        rng.integers(0, 5, size=(num_steps, num_worlds, 2))], axis=-1)
        return {
            "reset": (rng.random((num_steps, num_worlds, 1)) < 0.005).astype(np.int32),
            "action": act.astype(np.int32),
        }
    if sim == "arena":
        shape = (num_steps, num_worlds, 6)
        amount = np.where(rng.random(shape) < 0.6, 3, rng.integers(0, 4, size=shape))
        angle = np.where(rng.random(shape) < 0.6, 0, rng.integers(0, 8, size=shape))
        act = np.stack([amount, angle, rng.integers(0, 5, size=shape),
                        (rng.random(shape) < 0.15).astype(np.int64)], axis=-1)
        return {
            "reset": (rng.random((num_steps, num_worlds, 1)) < 0.004).astype(np.int32),
            "action": act.astype(np.int32),
        }
    if sim in ("balls", "balls_many", "hullpile", "hullpile_many"):
        return {}          # physics only: no inputs
    raise KeyError(sim)


def rollout_gpu(sim: str, num_worlds: int, num_steps: int, inputs, cfg=None, gpu_id: int = 0):
    """Roll a fixture sim on the GPU engine; returns outputs[name][steps+1, W, ...]."""
    import torch

    desc = SIMS[sim]
    ex = make_executor(sim, num_worlds, gpu_id=gpu_id, **(cfg or {}))
    graph = ex.buildLaunchGraphAllTaskGraphs()
    in_t = {s.name: ex.tensor(s.slot, s.dtype, (num_worlds,) + s.per_world) for s in desc.inputs}
    out_t = {s.name: ex.tensor(s.slot, s.dtype, (num_worlds,) + s.per_world)
             for s in desc.outputs if not s.dynamic}

    def grab(frames):
        for s in desc.outputs:
            if s.dynamic:
                rows = ex.exportedNumRows(s.slot)
                t = ex.tensor(s.slot, s.dtype, (max(rows, 1),) + s.per_world)
                frames[s.name].append(t.cpu().numpy()[:rows].copy())
            else:
                frames[s.name].append(out_t[s.name].cpu().numpy().copy())

    frames = {s.name: [] for s in desc.outputs}
    grab(frames)
    for step in range(num_steps):
        if inputs is not None:
            for s in desc.inputs:
                in_t[s.name].copy_(torch.from_numpy(np.ascontiguousarray(inputs[s.name][step])))
            torch.cuda.synchronize()
        ex.run(graph)
        grab(frames)
    n_kernels = graph.num_kernels
    del graph
    ex.close()
    dyn = {s.name for s in desc.outputs if s.dynamic}
    return {k: (v if k in dyn else np.stack(v)) for k, v in frames.items()}, n_kernels


def save_golden(name, inputs, outs, W, steps):
    payload = {"in_" + k: v for k, v in inputs.items()}
    for k, v in outs.items():
        if isinstance(v, list):
            payload["dyn_" + k] = np.concatenate(v) if v else np.zeros((0,))
            payload["dynlen_" + k] = np.array([len(f) for f in v], dtype=np.int64)
        else:
            payload["out_" + k] = v
    payload["meta"] = np.array([W, steps], dtype=np.int64)
    np.savez_compressed(golden_path(name), **payload)


def load_golden(name):
    z = np.load(golden_path(name))
    ins = {k[3:]: z[k] for k in z.files if k.startswith("in_")}
    outs = {k[4:]: z[k] for k in z.files if k.startswith("out_")}
    for k in z.files:
        if k.startswith("dyn_"):
            lens = z["dynlen_" + k[4:]]
            offs = np.concatenate([[0], np.cumsum(lens)])
            outs[k[4:]] = [z[k][offs[i]:offs[i + 1]] for i in range(len(lens))]
    W, steps = (int(v) for v in z["meta"])
    return W, steps, ins, outs


def assert_traces_equal(got, want, exact=True, rtol=1e-4, atol=1e-6):
    for k, w in want.items():
        g = got[k]
        if isinstance(w, list):
            assert len(g) == len(w), k
            for t, (gf, wf) in enumerate(zip(g, w)):
                assert gf.shape == wf.shape, f"{k} frame {t}: rows {gf.shape} vs {wf.shape}"
                assert np.array_equal(gf, wf), f"{k} frame {t} differs"
        elif exact or not np.issubdtype(w.dtype, np.floating):
            same = g.view(np.uint8) == w.view(np.uint8) if g.dtype.itemsize == 1 else g == w
            if np.issubdtype(w.dtype, np.floating):
                same = g.view(np.uint32) == w.view(np.uint32)
            assert same.all(), f"{k}: first mismatch at {np.argwhere(~same)[0]}"
        else:
            np.testing.assert_allclose(g, w, rtol=rtol, atol=atol, err_msg=k)


def golden_path(name: str) -> str:
    return os.path.join(GOLDEN_DIR, name + ".npz")


# Roll-outs too large to store as golden traces.  The reference CPU backend's trace of each
# is kept as one SHA-256 per exported column (written by tests/golden/make_golden.py), and
# the GPU trace must hash to the same value: a bit-exact comparison without the reference.
# name -> (sim, worlds, steps, seed of make_inputs (None: the sim has no inputs), sim cfg)
REFERENCE_CASES = {
    "cartpole_w256_s1000": ("cartpole", 256, 1000, 42, {}),
    "gridworld_w3000_s120": ("gridworld", 3000, 120, 77,
                             {"grid_size": 5, "episode_len": 30, "init_items": 10, "seed": 5}),
    "gridworld_w128_s60": ("gridworld", 128, 60, 13,
                           {"grid_size": 6, "episode_len": 25, "init_items": 8, "seed": 3}),
    "room_w300_s130": ("room", 300, 130, 9, {"episode_len": 60, "seed": 1000}),
    "room_grab_w200_s90": ("room", 200, 90, 4, {"episode_len": 50, "seed": 77, "grab_period": 3}),
    "room_w64_s60": ("room", 64, 60, 31, {"episode_len": 40, "seed": 7}),
    "room_tgs_w120_s50": ("room_tgs", 120, 50, 6, {"episode_len": 25, "seed": 300}),
    "arena_w160_s150": ("arena", 160, 150, 21, {"episode_len": 60, "seed": 4000}),
    "arena_w48_s70": ("arena", 48, 70, 77, {"episode_len": 45, "seed": 11}),
    "balls_w400_s150": ("balls", 400, 150, None, {"seed": 7000}),
    "balls_many_w48_s80": ("balls_many", 48, 80, None, {"seed": 31000}),
    "hullpile_w300_s120": ("hullpile", 300, 120, None, {"seed": 52000}),
    "hullpile_many_w48_s100": ("hullpile_many", 48, 100, None, {"seed": 53000}),
    "hullpile_w64_s60": ("hullpile", 64, 60, None, {"seed": 54000}),
}
# checked on the first worlds of a larger GPU run (tests/test_full_size.py, tests/test_hullpile.py)
PREFIX_CASES = {"gridworld_w128_s60", "room_w64_s60", "arena_w48_s70", "hullpile_w64_s60"}
DIGESTS_PATH = os.path.join(GOLDEN_DIR, "reference_digests.json")


def reference_case(name):
    """(sim, worlds, steps, inputs, cfg) of a REFERENCE_CASES entry."""
    sim, W, steps, seed, cfg = REFERENCE_CASES[name]
    ins = make_inputs(sim, W, steps, seed=seed) if seed is not None else {}
    return sim, W, steps, ins, dict(cfg)


def trace_digests(outs) -> Dict[str, str]:
    """SHA-256 of every column of a trace (shape and bytes of each frame)."""
    digests = {}
    for k, v in sorted(outs.items()):
        h = hashlib.sha256()
        for frame in (v if isinstance(v, list) else [v]):
            a = np.ascontiguousarray(frame)
            h.update(repr(a.shape).encode())
            h.update(a.tobytes())
        digests[k] = h.hexdigest()
    return digests


def reference_columns(name, outs):
    """The columns of a reference trace that the GPU test of `name` compares: the cases of
    PREFIX_CASES roll out only the fixed-size columns, and no entity handles (they come
    from one pool for all worlds, so they depend on the number of worlds)."""
    if name not in PREFIX_CASES:
        return dict(outs)
    dynamic = {s.name for s in SIMS[REFERENCE_CASES[name][0]].outputs if s.dynamic}
    return {k: v for k, v in outs.items() if k not in dynamic and not k.endswith("entity")}


def assert_matches_reference(name, got, exact=True, rtol=1e-4, atol=1e-5):
    """`got` has exactly the reference CPU backend's columns of REFERENCE_CASES[name], equal
    bit for bit (exact) or within rtol / atol on floats (a build with FMA contraction; this
    needs a live run of the reference, so it is skipped where oracle/_ref is not built)."""
    if not exact:
        import pytest
        from oracle import runner
        sim, W, steps, ins, cfg = reference_case(name)
        if not runner.available(sim):
            pytest.skip("a tolerance comparison needs the reference CPU backend (oracle/_ref)")
        ref, _ = runner.run_reference(SIMS[sim], W, steps, ins, cfg, workers=4)
        ref = reference_columns(name, ref)
        assert sorted(got) == sorted(ref), f"{name}: columns {sorted(got)}, reference {sorted(ref)}"
        assert_traces_equal(got, ref, exact=False, rtol=rtol, atol=atol)
        return
    with open(DIGESTS_PATH) as f:
        want = json.load(f)[name]
    assert sorted(got) == sorted(want), f"{name}: columns {sorted(got)}, reference {sorted(want)}"
    have = trace_digests(got)
    differ = [k for k in sorted(got) if have[k] != want[k]]
    assert not differ, f"{name}: columns differ from the reference CPU backend: {differ}"
