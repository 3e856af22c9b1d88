"""The grouping and work split of the physics ray queries (madrona_b200/csrc/physics_rays.cu),
modelled in numpy: the per-world histogram, the one-block scan, the scatter of ray indices into
slots (in any arrival order, as the atomics hand them out), the lane-per-slot kernel for worlds
of up to 128 leaves and the block-per-world kernel for larger ones.  Every ray of a world in
range is traced exactly once, by the kernel its world's leaf count selects, in its own world,
and its result lands at its own index; a ray of a world out of range is answered once, with a
miss, by the counting pass."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = open(os.path.join(ROOT, "madrona_b200", "csrc", "physics_rays.cu")).read()


def _const(name):
    m = re.search(r"constexpr int " + name + r" = (\d+);", SRC)
    assert m, name
    return int(m.group(1))


THREADS = _const("kRayThreads")
SCAN_THREADS = _const("kRayScanThreads")
LARGE_THREADS = _const("kRayLargeThreads")
SMALL_LEAVES = 128           # kSmallWorldLeaves = kMinWorldBodiesCap


def model(world, leaves, large_path, large_blocks, rng):
    """Which (kernel, ray index, world) each trace runs, and which rays the counting pass
    answers with a miss."""
    W, n = len(leaves), len(world)
    grid = (n + THREADS - 1) // THREADS
    valid = (world >= 0) & (world < W)
    # count kernel
    counts = np.zeros(W, dtype=np.int64)
    misses = []
    for i in range(grid * THREADS):
        if i >= n:
            continue
        if valid[i]:
            counts[world[i]] += 1
        else:
            misses.append(i)
    # scan kernel: each of SCAN_THREADS threads sums a run of `per` worlds
    per = (W + SCAN_THREADS - 1) // SCAN_THREADS
    offsets = np.zeros(W + 1, dtype=np.int64)
    for tid in range(SCAN_THREADS):
        first, last = min(W, tid * per), min(W, tid * per + per)
        for w in range(first, last):
            offsets[w] = counts[:w].sum()
    offsets[W] = counts.sum()
    cursor = offsets[:W].copy()
    # scatter kernel: the atomics hand out slots in any order
    order = np.full(n, -1, dtype=np.int64)
    for i in rng.permutation(n):
        if valid[i]:
            order[cursor[world[i]]] = i
            cursor[world[i]] += 1
    traces = []
    # lane-per-slot kernel
    for slot in range(grid * THREADS):
        if slot < offsets[W]:
            i = order[slot]
            w = world[i]
            if not (large_path and leaves[w] > SMALL_LEAVES):
                traces.append(("small", i, w))
    # block-per-world kernel
    if large_path:
        blocks = min(large_blocks, W)
        for b in range(blocks):
            for w in range(b, W, blocks):
                first, count = offsets[w], offsets[w + 1] - offsets[w]
                if count == 0 or leaves[w] <= SMALL_LEAVES:
                    continue
                for base in range(0, count, LARGE_THREADS):
                    for tid in range(LARGE_THREADS):
                        r = base + tid
                        if r < count:
                            i = order[first + r]
                            traces.append(("large", i, world[i]))
    return traces, misses


def check(world, leaves, large_path=True, large_blocks=132, seed=0):
    world = np.asarray(world, dtype=np.int64)
    leaves = np.asarray(leaves, dtype=np.int64)
    traces, misses = model(world, leaves, large_path, large_blocks, np.random.default_rng(seed))
    W = len(leaves)
    valid = (world >= 0) & (world < W)
    traced = [i for _, i, _ in traces]
    assert sorted(traced) == list(np.flatnonzero(valid)), "every ray in range traced exactly once"
    assert sorted(misses) == list(np.flatnonzero(~valid))
    for kind, i, w in traces:
        assert w == world[i]
        assert kind == ("large" if large_path and leaves[w] > SMALL_LEAVES else "small")
    return traces


def test_empty_and_single_ray():
    assert check([], [10, 200]) == []
    assert check([1], [10, 200]) == [("large", 0, 1)]
    assert check([0], [10, 200]) == [("small", 0, 0)]


def test_all_rays_in_one_world():
    rng = np.random.default_rng(1)
    for leaves in (5, 128, 129, 4096):
        check(np.full(1000, 3), rng.integers(1, 60, size=7).tolist()[:3] + [leaves] + [1, 2, 3])


def test_every_world_with_repeats_and_empty_worlds():
    rng = np.random.default_rng(2)
    W = 300
    leaves = rng.choice([0, 8, 128, 129, 500, 4096], size=W)
    world = rng.integers(0, W, size=5000)
    world = world[world % 7 != 0]                 # worlds w % 7 == 0 get no rays
    check(np.concatenate([world, world[:100]]), leaves)
    check(np.arange(W), leaves)                   # one ray per world


@pytest.mark.parametrize("n", [THREADS - 1, THREADS, THREADS + 1, 2 * THREADS + 1])
def test_block_edges(n):
    rng = np.random.default_rng(n)
    leaves = [20, 129, 3000, 0]
    check(rng.integers(0, 4, size=n), leaves)
    # a large world's rays across the block's round edges
    check(np.full(n, 1), leaves)


def test_large_path_off_traces_every_world_by_lane():
    rng = np.random.default_rng(3)
    leaves = [20, 129, 3000]
    traces = check(rng.integers(0, 3, size=700), leaves, large_path=False)
    assert {k for k, _, _ in traces} == {"small"}


def test_more_worlds_than_large_blocks_and_scan_threads():
    rng = np.random.default_rng(4)
    W = SCAN_THREADS + 77                          # several worlds per scan thread
    leaves = rng.choice([10, 200], size=W)
    check(rng.integers(0, W, size=3000), leaves, large_blocks=5)


def test_worlds_out_of_range_are_misses():
    check([0, 2, -1, 5, 1, 1 << 30, 2], [10, 200, 30])


def build_facade(tmp_path):
    """tests/cpp/facade_physics_rays.cpp, compiled and linked against the library."""
    import subprocess
    exe = str(tmp_path / "facade_physics_rays")
    cmd = ["g++", "-std=c++20", "-O1", "-I" + os.path.join(ROOT, "madrona_b200", "host"),
           os.path.join(ROOT, "tests", "cpp", "facade_physics_rays.cpp"), "-o", exe,
           "-L" + os.path.join(ROOT, "madrona_b200"), "-lmadrona_b200",
           "-Wl,-rpath," + os.path.join(ROOT, "madrona_b200"), "-L/usr/local/cuda/lib64", "-lcudart"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    return exe


def test_abi_layouts_and_facade_compile(tmp_path):
    """The Python records match the C structs, and the C++ facade program compiles and links."""
    import ctypes
    from madrona_b200.executor import _PhysicsRayHitsC, _PhysicsRaysC
    assert ctypes.sizeof(_PhysicsRaysC) == 32 and ctypes.sizeof(_PhysicsRayHitsC) == 24
    build_facade(tmp_path)


def test_null_executor_or_rays_are_rejected():
    import ctypes
    import madrona_b200 as mb
    from madrona_b200.executor import _PhysicsRayHitsC, _PhysicsRaysC, _last_error
    lib = mb.load_library()
    rays = _PhysicsRaysC(4, 4, 4, None)
    hits = _PhysicsRayHitsC(4, None, None)
    assert lib.mb2_trace_physics_rays(None, ctypes.byref(rays), 1, ctypes.byref(hits), None) == 1
    assert "mb2_trace_physics_rays: null executor or rays" in _last_error(lib)


def _golden():
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from trace_utils import load_golden
    return load_golden("rays_w1_s30")


def test_golden_covers_the_ray_mix():
    """The reference's one-world roll-out has what the fixture was built to exercise."""
    W, steps, _, outs = _golden()
    d, o, m = outs["ray_dir"][1:], outs["ray_origin"][1:], outs["ray_max_t"][1:]
    hit = outs["hit_entity"][1:, ..., 1] >= 0
    assert hit.any() and (~hit).any()
    assert (np.signbit(d) & (d == 0)).any()                   # -0.f components
    assert ((np.abs(d) == 1).sum(-1) == 1).any()              # axis-aligned rays
    assert (o[..., 2] < 0).any() and (d[..., 2] == 0).any()   # from below / parallel to the plane
    assert np.isinf(m).any() and (np.isfinite(m) & (m < 1)).any()
    assert (outs["hit_t"][1:][hit] >= 0).all()
    n = np.linalg.norm(outs["hit_normal"][1:][hit], axis=-1)
    assert np.allclose(n, 1, atol=1e-4)
    assert len(set(outs["body_count"][:, 0, 0].tolist())) >= 3    # respawns at other sizes


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "ref_rays")),
                    reason="the reference CPU backend is not built here (oracle/rays.mk)")
def test_reference_reproduces_the_digests():
    import json
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from oracle.runner import run_reference
    from sims import SIMS
    from test_physics_rays import RAYS_DIGESTS_PATH, RAYS_REFERENCE_CASES
    from trace_utils import trace_digests
    want = json.load(open(RAYS_DIGESTS_PATH))
    assert sorted(want) == sorted(RAYS_REFERENCE_CASES)
    for case, (W, steps, cfg, _) in RAYS_REFERENCE_CASES.items():
        assert trace_digests(run_reference(SIMS["rays"], W, steps, {}, cfg, workers=2)[0]) == want[case], case
