"""Physics ray queries (mb2_trace_physics_rays / MWCudaExecutor.tracePhysicsRays) against the
simulator's own BVH::traceRay.  The rays fixture (sims/rays) fills 64 rays per world before
physics and traces them in its last node; the same rays, handed to the engine after the step
as one shuffled batch with repeats, must give the exported hits byte for byte -- on worlds of
8 to 60 bodies, of 129, 1024 and 4096 bodies (MADRONA_B200_MAX_BODIES_PER_WORLD, the
block-per-world path with the boxes in shared memory) and with spheres among the bodies.
The same rays in world order, every frame, must also hash to the reference CPU backend's
traceRay hits (tests/golden/rays_digests.json, written by tests/golden/make_rays_golden.py),
independently of the shared source.  Further: a batch with worlds on both sides of 128 leaves,
the C++ facade, no side effect on the simulation, caller streams, snapshots, the first step,
rejected calls and rays of worlds out of range."""
import ctypes
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

EXACT = os.environ.get("MADRONA_B200_FAST_MATH", "0") != "1"
K = 64              # rays per world (sims/rays kRaysPerWorld)
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RAYS_DIGESTS_PATH = os.path.join(GOLDEN_DIR, "rays_digests.json")
KNOB = "MADRONA_B200_MAX_BODIES_PER_WORLD"

# Roll-outs of sims/rays on the reference CPU backend, kept as one SHA-256 per exported column
# (tests/golden/make_rays_golden.py); rays_w1_s30 is also kept whole as a golden npz.  The
# hits of each frame are the reference's traceRay; the engine's world-major batch of the same
# rays must hash the same.  Worlds respawn (episode_len > 0) only in the one-world case: the
# handles of respawned bodies come from one pool for all worlds, handed out in another order by
# each backend.  name -> (worlds, steps, cfg, MADRONA_B200_MAX_BODIES_PER_WORLD or None)
RAYS_REFERENCE_CASES = {
    # resets every 7 steps: the trees are rebuilt, at 55, 15 and 40 bodies
    "rays_w1_s30": (1, 30, {"seed": 3, "episode_len": 7}, None),
    # 32 worlds of 8 to 60 bodies
    "rays_w32_s20": (32, 20, {"seed": 40, "episode_len": 0}, None),
    # worlds of 8 to 300 bodies in one batch: both trace kernels have work in every call
    "rays_mixed_w24_s12": (24, 12, {"seed": 7, "episode_len": 0, "varied_bodies": 300}, "512"),
    # every world past 128 leaves: the block-per-world kernel with the boxes in shared memory
    "rays_b129_w8_s12": (8, 12, {"seed": 11, "episode_len": 0, "uniform_bodies": 129}, "129"),
    "rays_b1024_w2_s10": (2, 10, {"seed": 11, "episode_len": 0, "uniform_bodies": 1024}, "1024"),
    "rays_b4096_w1_s8": (1, 8, {"seed": 11, "episode_len": 0, "uniform_bodies": 4096}, "4096"),
}
RAYS_GOLDEN = "rays_w1_s30"


def _make(sim="rays", W=16, **cfg):
    from sims import make_executor
    return make_executor(sim, W, **cfg)


def _fixture_rays(ex, W):
    """The step's rays and the in-simulator hits, world-major, as GPU tensors."""
    import torch
    flat = lambda slot, dt, shape: ex.tensor(slot, dt, (W, K) + shape).reshape((W * K,) + shape)
    world = torch.arange(W, dtype=torch.int32, device="cuda").repeat_interleave(K)
    return (world, flat(0, "float32", (3,)).clone(), flat(1, "float32", (3,)).clone(),
            flat(2, "float32", ()).clone(),
            {"entity": flat(3, "int32", (2,)).clone(), "t": flat(4, "float32", ()).clone(),
             "normal": flat(5, "float32", (3,)).clone()})


def _shuffled_with_repeats(n, gen):
    import torch
    idx = torch.cat([torch.randperm(n, generator=gen), torch.randint(0, n, (n // 2 + 1,), generator=gen)])
    return idx[torch.randperm(len(idx), generator=gen)].cuda()


def _assert_same(got, want, what=""):
    for k, w in want.items():
        g = got[k]
        assert g.shape == w.shape, (what, k)
        if EXACT or k == "entity":
            same = g.view(torch_int32()) == w.view(torch_int32())
            assert bool(same.all()), f"{what} {k}: {int((~same).sum())} values differ"
        else:
            np.testing.assert_allclose(g.cpu().numpy(), w.cpu().numpy(), rtol=1e-4, atol=1e-5)


def torch_int32():
    import torch
    return torch.int32


def _roll_and_check(ex, W, steps, seed=0):
    """Every step: the fixture's rays as a shuffled batch with repeats give its hits; in world
    order, without max_t where it is +inf everywhere, they give them too.  Returns the number
    of hits and misses seen."""
    import torch
    gen = torch.Generator().manual_seed(seed)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    hits = misses = 0
    for step in range(steps):
        ex.run(graph)
        world, o, d, m, want = _fixture_rays(ex, W)
        idx = _shuffled_with_repeats(W * K, gen)
        got = ex.tracePhysicsRays(world[idx], o[idx], d[idx], m[idx])
        _assert_same(got, {k: v[idx] for k, v in want.items()}, f"step {step} shuffled")
        got = ex.tracePhysicsRays(world, o, d, m)
        _assert_same(got, want, f"step {step} world-major")
        hit = want["entity"][:, 1] >= 0
        hits += int(hit.sum())
        misses += int((~hit).sum())
    del graph
    return hits, misses


def test_batches_match_in_simulator_trace_ray():
    ex = _make("rays", 48, seed=3, episode_len=7)
    hits, misses = _roll_and_check(ex, 48, 20)
    assert hits > 1000 and misses > 100
    ex.close()


def _uniform_env(monkeypatch, bodies):
    for k, v in {"MADRONA_B200_ROWS_PER_WORLD": str(bodies), "MADRONA_B200_PERSIST_BYTES": str(512 << 20),
                 "MADRONA_B200_MAX_CANDIDATES_PER_WORLD": str(16 * bodies),
                 "MADRONA_B200_MAX_CONTACTS_PER_WORLD": str(8 * bodies),
                 "MADRONA_B200_MAX_BODIES_PER_WORLD": str(bodies)}.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("bodies,W", [(129, 40), (1024, 4), (4096, 2)])
def test_large_worlds_match_in_simulator_trace_ray(monkeypatch, bodies, W):
    _uniform_env(monkeypatch, bodies)
    ex = _make("rays", W, seed=11, episode_len=0, uniform_bodies=bodies)
    hits, misses = _roll_and_check(ex, W, 8, seed=bodies)
    assert hits > 0 and misses > 0
    ex.close()


def test_large_and_small_worlds_in_one_batch(monkeypatch):
    # worlds of 8 to 300 bodies, respawning at other sizes: every call gives the lane-per-ray
    # kernel the worlds of up to 128 leaves and the block-per-world kernel the others
    _uniform_env(monkeypatch, 512)
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "1024")    # old and new bodies until compaction
    ex = _make("rays", 24, seed=5, episode_len=5, varied_bodies=300)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(12):
        ex.run(graph)
        counts = ex.tensor(6, "int32", (24,))
        assert bool((counts > 128).any()) and bool((counts <= 128).any())
    del graph
    hits, misses = _roll_and_check(ex, 24, 12, seed=5)
    assert hits > 0 and misses > 0
    ex.close()


def _reference_env(monkeypatch, case):
    W, steps, cfg, knob = RAYS_REFERENCE_CASES[case]
    if knob is not None:
        _uniform_env(monkeypatch, int(knob))


def rollout_world_major(ex, W, steps):
    """The fixture's columns of every frame, with the hit columns from the engine's world-major
    batch of the frame's rays (frame 0: before the first step) instead of the simulator's."""
    from sims import SIMS
    outs = {s.name: [] for s in SIMS["rays"].outputs}
    graph = ex.buildLaunchGraphAllTaskGraphs()
    for step in range(steps + 1):
        if step > 0:
            ex.run(graph)
        world, o, d, m, _ = _fixture_rays(ex, W)
        hits = ex.tracePhysicsRays(world, o, d, m)
        outs["ray_origin"].append(o.view(W, K, 3).cpu().numpy())
        outs["ray_dir"].append(d.view(W, K, 3).cpu().numpy())
        outs["ray_max_t"].append(m.view(W, K).cpu().numpy())
        outs["hit_entity"].append(hits["entity"].view(W, K, 2).cpu().numpy())
        outs["hit_t"].append(hits["t"].view(W, K).cpu().numpy())
        outs["hit_normal"].append(hits["normal"].view(W, K, 3).cpu().numpy())
        outs["body_count"].append(ex.tensor(6, "int32", (W, 1)).cpu().numpy())
        rows = ex.exportedNumRows(7)
        outs["body_pos"].append(ex.tensor(7, "float32", (max(rows, 1), 3)).cpu().numpy()[:rows].copy())
        outs["body_entity"].append(ex.tensor(8, "int32", (max(rows, 1), 2)).cpu().numpy()[:rows].copy())
    del graph
    dyn = {"body_pos", "body_entity"}
    return {k: (v if k in dyn else np.stack(v)) for k, v in outs.items()}


@pytest.mark.parametrize("case", sorted(RAYS_REFERENCE_CASES))
def test_world_major_batches_match_the_reference(monkeypatch, case):
    """Every frame's hits from the engine, world-major, hash to the reference CPU backend's
    traceRay hits of the same rays, and the rest of the roll-out to the reference's columns."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from trace_utils import trace_digests
    if not EXACT:
        pytest.skip("the digests are bit-exact; a build with FMA contraction rounds differently")
    _reference_env(monkeypatch, case)
    W, steps, cfg, _ = RAYS_REFERENCE_CASES[case]
    ex = _make("rays", W, **cfg)
    got = rollout_world_major(ex, W, steps)
    ex.close()
    with open(RAYS_DIGESTS_PATH) as f:
        want = json.load(f)[case]
    have = trace_digests(got)
    assert sorted(have) == sorted(want)
    differ = [k for k in sorted(want) if have[k] != want[k]]
    assert not differ, f"{case}: columns differ from the reference CPU backend: {differ}"


def test_spheres_are_skipped_like_trace_ray():
    ex = _make("rays_spheres", 32, seed=9, episode_len=9)
    hits, _ = _roll_and_check(ex, 32, 15)
    assert hits > 0
    ex.close()


def test_calls_change_nothing():
    import torch
    a = _make("rays", 16, seed=21, episode_len=6)
    b = _make("rays", 16, seed=21, episode_len=6)
    ga, gb = a.buildLaunchGraphAllTaskGraphs(), b.buildLaunchGraphAllTaskGraphs()
    cols = [(0, "float32", 3), (1, "float32", 3), (2, "float32", 1), (3, "int32", 2), (4, "float32", 1),
            (5, "float32", 3)]
    for step in range(14):
        a.run(ga)
        b.run(gb)
        world, o, d, m, _ = _fixture_rays(a, 16)
        before = [a.tensor(s, dt, (16 * K, c)).clone() for s, dt, c in cols]
        for _ in range(3):
            a.tracePhysicsRays(world, o, d, m)
        for (s, dt, c), x in zip(cols, before):
            assert torch.equal(a.tensor(s, dt, (16 * K, c)), x)
            assert torch.equal(b.tensor(s, dt, (16 * K, c)), x), f"step {step} slot {s}"
        na, nb = a.exportedNumRows(7), b.exportedNumRows(7)
        assert na == nb
        assert torch.equal(a.tensor(7, "float32", (na, 3)), b.tensor(7, "float32", (nb, 3)))
    del ga, gb
    a.close()
    b.close()


def test_caller_stream_equals_synchronous_call():
    import torch
    ex = _make("rays", 32, seed=2)
    g = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(4):
        ex.run(g)
    world, o, d, m, want = _fixture_rays(ex, 32)
    sync = ex.tracePhysicsRays(world, o, d, m)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = ex.tracePhysicsRays(world, o, d, m, stream=s)
    s.synchronize()
    for k in sync:
        assert torch.equal(got[k], sync[k])
    _assert_same(sync, want)
    del g
    ex.close()


def test_snapshot_restore_gives_the_saved_trees():
    import torch
    ex = _make("rays", 16, seed=4, episode_len=5)
    g = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(3):
        ex.run(g)
    snap = ex.snapshot()
    snap.save()
    world, o, d, m, want = _fixture_rays(ex, 16)
    at_save = ex.tracePhysicsRays(world, o, d, m)
    _assert_same(at_save, want)
    for _ in range(4):            # past an episode reset: the trees are rebuilt
        ex.run(g)
    moved = ex.tracePhysicsRays(world, o, d, m)
    assert not all(torch.equal(moved[k], at_save[k]) for k in moved)
    snap.restore()
    torch.cuda.synchronize()
    restored = ex.tracePhysicsRays(world, o, d, m)
    for k in at_save:
        assert torch.equal(restored[k], at_save[k])
    snap.close()
    del g
    ex.close()


def test_every_ray_misses_before_the_first_step():
    import torch
    ex = _make("rays", 8, seed=1)
    n = 500
    gen = torch.Generator().manual_seed(0)
    world = torch.randint(0, 8, (n,), generator=gen)
    o = torch.rand((n, 3), generator=gen) * 8 - 4
    d = torch.rand((n, 3), generator=gen) * 2 - 1
    got = ex.tracePhysicsRays(world, o, d)
    assert (got["entity"] == torch.tensor([-1, -1], dtype=torch.int32, device="cuda")).all()
    assert (got["t"] == 0).all() and (got["normal"] == 0).all()
    ex.close()


def test_facade_matches_python_call(tmp_path):
    """tests/cpp/facade_physics_rays.cpp: the fixture's rays, reversed, after 5 steps of 4 worlds
    (seeds 5 - 8, a respawn every 4 steps), through MWCudaExecutor::tracePhysicsRays."""
    import subprocess
    import sys
    import torch
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from sims import SIMS
    from sims.objects import write_blob_file
    from test_physics_rays_model import build_facade
    exe = build_facade(tmp_path)
    objects, out = str(tmp_path / "objects.bin"), str(tmp_path / "hits.bin")
    write_blob_file(objects, *SIMS["rays"].objects())
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([exe, os.path.join(root, "sims", "rays", "sim.cpp"), objects, out],
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    raw = np.fromfile(out, dtype=np.uint8)
    W = 4
    n = W * K
    assert raw.size == n * 24
    ex = _make("rays", W, seed=5, episode_len=4)
    g = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(5):
        ex.run(g)
    world, o, d, m, want = _fixture_rays(ex, W)
    rev = torch.arange(n - 1, -1, -1, device="cuda")
    got = ex.tracePhysicsRays(world[rev], o[rev], d[rev], m[rev])
    _assert_same(got, {k: v[rev] for k, v in want.items()})
    del g
    ex.close()
    parts = [got[k].cpu().numpy().reshape(-1).view(np.uint8) for k in ("entity", "t", "normal")]
    assert np.array_equal(raw, np.concatenate(parts))


def _raw_call(ex, rays, n, hits):
    import madrona_b200.executor as mbe
    r = mbe._PhysicsRaysC(*rays) if rays is not None else None
    h = mbe._PhysicsRayHitsC(*hits)
    rc = ex._lib.mb2_trace_physics_rays(ex._h if ex is not None else None,
                                        ctypes.byref(r) if r is not None else None, n, ctypes.byref(h), None)
    return rc, mbe._last_error(ex._lib) if rc else ""


def test_rejected_calls_launch_nothing():
    import torch
    import madrona_b200 as mb
    ex = _make("rays", 4, seed=1)
    g = ex.buildLaunchGraphAllTaskGraphs()
    ex.run(g)
    world, o, d, m, _ = _fixture_rays(ex, 4)
    n = 4 * K
    ent = torch.full((n + 1, 2), 7, dtype=torch.int32, device="cuda")
    t = torch.full((n + 1,), 7.0, device="cuda")
    nrm = torch.full((n + 1, 3), 7.0, device="cuda")
    rays = (world.data_ptr(), o.data_ptr(), d.data_ptr(), m.data_ptr())
    hits = (ent.data_ptr(), t.data_ptr(), nrm.data_ptr())

    def untouched():
        torch.cuda.synchronize()
        return bool((ent == 7).all() and (t == 7).all() and (nrm == 7).all())

    cases = [
        ("null rays", lambda: _raw_call(ex, None, n, hits), "null executor or rays"),
        ("no output", lambda: _raw_call(ex, rays, n, (None, None, None)), "every output"),
        ("null origin", lambda: _raw_call(ex, (rays[0], None, rays[2], rays[3]), n, hits), "must not be NULL"),
        ("misaligned t", lambda: _raw_call(ex, rays, n, (hits[0], hits[1] + 2, hits[2])), "t is not 4-byte aligned"),
        ("misaligned origin", lambda: _raw_call(ex, (rays[0], rays[1] + 1, rays[2], rays[3]), n, hits),
         "origin is not 4-byte aligned"),
        ("misaligned max_t", lambda: _raw_call(ex, rays[:3] + (rays[3] + 2,), n, hits), "max_t is not"),
    ]
    for name, call, msg in cases:
        rc, err = call()
        assert rc == 1 and msg in err, (name, err)
        assert untouched(), name
    lib = ex._lib
    h = __import__("madrona_b200.executor", fromlist=["x"])._PhysicsRayHitsC(*hits)
    assert lib.mb2_trace_physics_rays(None, None, n, ctypes.byref(h), None) == 1
    # n = 0: a successful no-op, with or without pointers
    assert _raw_call(ex, rays, 0, hits)[0] == 0
    assert _raw_call(ex, (None, None, None, None), 0, (None, None, None))[0] == 0
    assert untouched()
    out = ex.tracePhysicsRays(world[:0], o[:0], d[:0])
    assert out["entity"].shape == (0, 2) and out["t"].shape == (0,) and out["normal"].shape == (0, 3)
    with pytest.raises(mb.MadronaB200Error, match="every output"):
        ex.tracePhysicsRays(world, o, d, entity=False, t=False, normal=False)
    ex.run(g)                       # the executor is still fine
    del g
    ex.close()

    # a simulator without PhysicsSystem
    cart = _make("cartpole", 4)
    with pytest.raises(mb.MadronaB200Error, match="PhysicsSystem::registerTypes"):
        cart.tracePhysicsRays(torch.zeros(3, dtype=torch.int32), torch.zeros(3, 3), torch.ones(3, 3))
    cart.close()


def test_out_of_range_world_misses_and_fails_the_next_run():
    import torch
    import madrona_b200 as mb
    ex = _make("rays", 6, seed=8)
    g = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(2):
        ex.run(g)
    world, o, d, m, want = _fixture_rays(ex, 6)
    w = world.clone()
    w[5] = 6
    w[K + 3] = -1
    w[2 * K] = 1 << 30
    got = ex.tracePhysicsRays(w, o, d, m)
    bad = torch.zeros(6 * K, dtype=torch.bool, device="cuda")
    bad[[5, K + 3, 2 * K]] = True
    assert (got["entity"][bad] == -1).all() and (got["t"][bad] == 0).all() and (got["normal"][bad] == 0).all()
    _assert_same({k: v[~bad] for k, v in got.items()}, {k: v[~bad] for k, v in want.items()})
    with pytest.raises(mb.MadronaB200Error, match="physics ray query with a world outside"):
        ex.run(g)
    del g
    ex.close()
    torch.cuda.synchronize()
    assert torch.arange(1024, device="cuda").sum().item() == 1023 * 512
