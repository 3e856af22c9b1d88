"""Navigation meshes (<madrona/navmesh.hpp>, <madrona/memory.hpp>, the new <madrona/utils.hpp>
names) and the host navmesh builder (mb2_navmesh_create / madrona_b200.Navmesh).

* oracle/navmesh_probe.cpp, built against the reference and against the engine's headers,
  must print the same arrays, samples, BFS / Dijkstra visit sequences and utils results.
* sims/navmesh runs on the reference CPU backend (every world builds its own navmesh in its
  constructor; one more is shared through Config); its trace is kept as a golden
  (navmesh_w9_s60.npz) and as per-column digests of larger roll-outs (navmesh_digests.json),
  both written by tests/golden/make_navmesh_golden.py.  The GPU engine must reproduce them
  bit for bit."""
import json
import os
import subprocess

import numpy as np
import pytest

from trace_utils import GOLDEN_DIR, assert_traces_equal, load_golden, rollout_gpu, trace_digests

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
FLT_MAX = np.float32(3.4028235e38)
SENTINEL = 0xFFFFFFFF
NUM_AGENTS = 6

# golden -> (worlds, steps, sim cfg)
GOLDENS = {"navmesh_w9_s60": (9, 60, {"seed": 5, "episode_len": 23})}
# case -> (worlds, steps, sim cfg); the 8192-world case is the first steps of a full-size run
DIGEST_CASES = {
    "navmesh_w300_s60": (300, 60, {"seed": 300, "episode_len": 25}),
    "navmesh_shared_w64_s40": (64, 40, {"seed": 77, "episode_len": 15, "per_world": False}),
    "navmesh_w8192_s12": (8192, 12, {"seed": 9000, "episode_len": 7}),
}
DIGESTS_PATH = os.path.join(GOLDEN_DIR, "navmesh_digests.json")


def _digests():
    with open(DIGESTS_PATH) as f:
        return json.load(f)


def _probe(which):
    exe = os.path.join(REF_DIR, f"navmesh_probe_{which}")
    if not os.path.exists(exe):
        pytest.skip(f"needs {exe} (make -C oracle -f navmesh.mk navmesh)")
    return subprocess.run([exe], check=True, capture_output=True, text=True).stdout


def _probe_soups(text):
    """soup name -> (V, T, vertex lines, triangle lines)"""
    soups, cur = {}, None
    for line in text.splitlines():
        if line.startswith("soup "):
            _, name, _, v, _, t = line.split()
            cur = soups[name] = (int(v), int(t), [], [])
        elif cur is not None and line.startswith("v "):
            cur[2].append(line)
        elif cur is not None and line.startswith("t "):
            cur[3].append(line)
    return soups


def _mesh_from_probe_lines(tri_lines):
    idx, adj, tau, alias = [], [], [], []
    for line in tri_lines:
        a, b, c = line[2:].split(" | ")
        idx.append([int(x) for x in a.split()])
        adj.append([int(x) for x in b.split()])
        t, al = c.split()
        tau.append(int(t, 16))
        alias.append(int(al))
    return (np.array(idx, np.uint32), np.array(adj, np.uint32), np.array(tau, np.uint32).view(np.float32),
            np.array(alias, np.uint32))


# ---- CPU: the engine's headers against the reference ---------------------------------------

def test_probe_matches_reference():
    ref, mine = _probe("ref"), _probe("mine")
    assert len(ref) > 1_000_000
    ref_lines, mine_lines = ref.splitlines(), mine.splitlines()
    assert len(ref_lines) == len(mine_lines)
    for i, (r, m) in enumerate(zip(ref_lines, mine_lines)):
        assert r == m, f"line {i}: {r[:200]!r} vs {m[:200]!r}"


def test_probe_exercises_the_feature():
    text = _probe("ref")
    soups = _probe_soups(text)
    assert {"single", "repeated", "zeroarea"} <= set(soups) and len(soups) > 25
    # a single triangle: a 1-slot ArrayQueue is empty as soon as it is filled, so BFS visits nothing
    assert "b 0:\n" in text.split("soup single")[1]
    # Dijkstra settles each triangle once
    for line in text.splitlines():
        if line.startswith("d "):
            visited = [int(x.split("/")[0]) for x in line.split(":")[1].split()]
            assert len(visited) == len(set(visited))
    assert "queue cap 5" in text and " c1" in text


def test_host_builder_matches_reference_probe():
    import madrona_b200 as mb
    from sims.navmesh_plan import SHARED_PLAN_SEED, make_plan
    soups = _probe_soups(_probe("ref"))
    for seed in [SHARED_PLAN_SEED] + list(range(12)):
        verts, polys = make_plan(seed)
        nm = mb.Navmesh(verts, polys, -1)
        a = nm.arrays()
        nm.close()
        V, T, vlines, tlines = soups[f"plan{seed}"]
        idx, adj, tau, alias = _mesh_from_probe_lines(tlines)
        assert (len(a["vertices"]), len(a["tri_indices"])) == (V, T)
        want_v = np.array([[int(x, 16) for x in line.split()[1:]] for line in vlines], np.uint32)
        assert (a["vertices"].view(np.uint32) == want_v).all()
        assert (a["tri_indices"] == idx).all() and (a["tri_adjacency"] == adj).all()
        assert (a["alias_tau"].view(np.uint32) == tau.view(np.uint32)).all() and (a["alias"] == alias).all()


def test_python_plan_matches_the_fixture_plan():
    from sims.navmesh_plan import SHARED_PLAN_SEED, make_plan
    text = _probe("ref")
    for seed in [SHARED_PLAN_SEED] + list(range(12)):
        head = f"plan {seed} V "
        block = text.split(head, 1)[1].splitlines()
        V, P, I = (int(x) for x in block[0].split()[::2])
        verts, polys = make_plan(seed)
        assert (len(verts), len(polys), sum(map(len, polys))) == (V, P, I)
        assert (verts.reshape(-1).view(np.uint32) == np.array([int(x, 16) for x in block[1].split()], np.uint32)).all()
        assert [int(x) for x in block[3].split()] == [v for p in polys for v in p]


def test_shared_plan_has_every_feature():
    import madrona_b200 as mb
    from sims.navmesh_plan import SHARED_PLAN_SEED, make_plan
    verts, polys = make_plan(SHARED_PLAN_SEED)
    assert {4, 5, 6, 3} <= {len(p) for p in polys}
    a = mb.Navmesh(verts, polys).arrays()
    T = len(a["tri_indices"])
    tri = verts[a["tri_indices"].astype(np.int64)]
    w = np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    assert (w == 0).any()                                     # the hexagon's first fan triangle
    assert w.sum() == T and (w == 1).sum() > T // 2           # unit weights normalise to exactly 1
    edges = {}
    for t, (x, y, z) in enumerate(a["tri_indices"]):
        for e in ((x, y), (y, z), (z, x)):
            edges.setdefault(tuple(sorted(e)), []).append(t)
    assert max(len(v) for v in edges.values()) == 3           # the fin's edge
    assert ((a["alias"] != np.arange(T)) & (a["alias_tau"] < 1)).any()
    # islands: the weight-2 triangles have no neighbours
    lonely = (a["tri_adjacency"] == SENTINEL).all(axis=1)
    assert lonely.sum() >= 1


def _decrease_key_events(a, start):
    """Dijkstra over the host arrays as navmesh.hpp runs it (float32, midpoints of edges
    (a,b) (b,c) (c,a)); counts relaxations of a triangle already in the queue."""
    import heapq
    v = a["vertices"]
    tri, adj = a["tri_indices"], a["tri_adjacency"]
    T = len(tri)
    dist = np.full(T, FLT_MAX, np.float32)
    entry = np.zeros((T, 3), np.float32)
    entry[start] = (v[tri[start, 0]] + v[tri[start, 1]] + v[tri[start, 2]]) / np.float32(3)
    dist[start] = 0
    queued, done, heap, events = {start}, set(), [(np.float32(0), start)], 0
    while heap:
        d, p = heapq.heappop(heap)
        if p in done or d != dist[p]:
            continue
        done.add(p)
        queued.discard(p)
        x = v[tri[p]]
        mids = [(x[0] + x[1]) * np.float32(0.5), (x[1] + x[2]) * np.float32(0.5), (x[2] + x[0]) * np.float32(0.5)]
        for i in range(3):
            n = int(adj[p, i])
            if n == SENTINEL:
                continue
            nd = np.float32(d + np.float32(np.sqrt(np.float32(((entry[p] - mids[i]) ** 2).sum()))))
            if nd >= dist[n]:
                continue
            events += n in queued
            dist[n], entry[n] = nd, mids[i]
            queued.add(n)
            heapq.heappush(heap, (nd, n))
    return events


def test_shared_plan_dijkstra_decreases_keys():
    import madrona_b200 as mb
    from sims.navmesh_plan import SHARED_PLAN_SEED, make_plan
    verts, polys = make_plan(SHARED_PLAN_SEED)
    a = mb.Navmesh(verts, polys).arrays()
    assert sum(_decrease_key_events(a, s) for s in range(len(a["tri_indices"]))) > 0


@pytest.mark.parametrize("bad, msg", [
    ("no_polys", "no polygons"),
    ("small", "at least 3"),
    ("past_end", "runs past the index array"),
    ("bad_index", "names vertex"),
])
def test_host_builder_rejects_bad_input(bad, msg):
    import madrona_b200 as mb
    verts = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32)
    polys = {
        "no_polys": [],
        "small": [[0, 1, 2], [2, 3]],
        "past_end": (np.array([0, 1, 2, 3], np.uint32), np.array([0, 2], np.uint32), np.array([4, 3], np.uint32)),
        "bad_index": [[0, 1, 2, 3], [0, 2, 7]],
    }[bad]
    with pytest.raises(mb.MadronaB200Error, match=msg):
        mb.Navmesh(verts, polys)


def test_host_builder_rejects_null_arrays():
    import madrona_b200 as mb
    lib = mb.load_library()
    assert not lib.mb2_navmesh_create(None, 3, None, 3, None, None, 1, -1)
    assert b"null input array" in lib.mb2_last_error()


def test_host_builder_view_needs_a_gpu():
    import madrona_b200 as mb
    nm = mb.Navmesh(np.eye(3, dtype=np.float32), [[0, 1, 2]])
    with pytest.raises(mb.MadronaB200Error, match="without a GPU"):
        nm.view_bytes()
    nm.close()


# ---- CPU: the golden exercises the feature --------------------------------------------------

def test_golden_exercises_the_feature():
    W, steps, _, outs = load_golden("navmesh_w9_s60")
    mesh = outs["mesh"][0]
    own_T, shared_T = mesh[:, 1], mesh[:, 4]
    assert (own_T > 0).all() and len(np.unique(mesh[:, 0])) == W and (shared_T == shared_T[0]).all()
    bfs = outs["bfs"][1:]
    T_of_agent = np.where(np.arange(NUM_AGENTS) % 2 == 1, shared_T[:, None], own_T[:, None])
    accepted, rejected = bfs[..., 0], bfs[..., 1]
    # islands: BFS reaches less than the mesh, and goals on another island stay at FLT_MAX
    assert (accepted + rejected < T_of_agent[None]).any()
    assert (outs["dist"][1:] == FLT_MAX).any() and (outs["dist"][1:] < 100).any()
    assert (rejected > 0).any()
    # Dijkstra stops at island borders; visit orders differ between agents and steps
    visits = outs["dijkstra"][1:, :, :, 0]
    assert (visits < T_of_agent[None]).any() and (visits <= T_of_agent[None]).all()
    assert len(np.unique(outs["dijkstra"][1:, :, :, 1])) > 200
    # agents move, reach goals and respawn
    pos = outs["pos"]
    assert (pos[1:] != pos[:-1]).any(axis=(1, 2, 3)).mean() > 0.9
    goals = outs["goal"]
    assert (goals[1:] != goals[:-1]).any(axis=3).sum() > W * NUM_AGENTS * 2


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_reference_reproduces_golden(name):
    from oracle import runner
    from sims import SIMS
    W, steps, cfg = GOLDENS[name]
    if not runner.available("navmesh"):
        pytest.skip("needs oracle/_ref/ref_navmesh (make -C oracle -f navmesh.mk navmesh)")
    _, _, _, want = load_golden(name)
    got, _ = runner.run_reference(SIMS["navmesh"], W, steps, None, cfg, workers=1)
    assert_traces_equal(got, want)


# ---- GPU: parity ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_matches_golden(name):
    W, steps, cfg = GOLDENS[name]
    _, _, _, want = load_golden(name)
    got, n_kernels = rollout_gpu("navmesh", W, steps, None, cfg)
    assert n_kernels > 0
    assert sorted(got) == sorted(want)
    assert_traces_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(DIGEST_CASES))
def test_matches_reference_digests(case):
    W, steps, cfg = DIGEST_CASES[case]
    got, _ = rollout_gpu("navmesh", W, steps, None, cfg)
    want = _digests()[case]
    have = trace_digests(got)
    assert sorted(have) == sorted(want)
    assert [k for k in sorted(want) if have[k] != want[k]] == []


@pytest.mark.gpu
def test_matches_live_reference():
    from oracle import runner
    from sims import SIMS
    if not runner.available("navmesh"):
        pytest.skip("needs oracle/_ref/ref_navmesh")
    W, steps, cfg = 37, 45, {"seed": 1234, "episode_len": 17}
    want, _ = runner.run_reference(SIMS["navmesh"], W, steps, None, cfg, workers=2)
    got, _ = rollout_gpu("navmesh", W, steps, None, cfg)
    assert_traces_equal(got, want)


@pytest.mark.gpu
def test_shared_navmesh_view_holds_device_pointers():
    import madrona_b200 as mb
    from sims.navmesh_plan import SHARED_PLAN_SEED, make_plan
    verts, polys = make_plan(SHARED_PLAN_SEED)
    nm = mb.Navmesh(verts, polys, 0)
    view = nm.view_bytes()
    ptrs = np.frombuffer(view[:32], np.uint64)
    nv, T = (int(x) for x in np.frombuffer(view[32:], np.uint32))
    a = nm.arrays()
    nm.close()
    assert (nv, T) == (len(verts), len(a["tri_indices"]))
    assert (ptrs != 0).all() and (ptrs % 256 == 0).all() and len(set(ptrs.tolist())) == 4


def _persist_need(mesh_info):
    r128 = lambda b: (b + 127) // 128 * 128
    T, V = mesh_info[:, 1].astype(np.int64), mesh_info[:, 2].astype(np.int64)
    return int(sum(r128(12 * v) + 2 * r128(12 * t) + r128(8 * t) for t, v in zip(T, V)))


@pytest.mark.gpu
def test_construction_under_table_growth_reclaims_persistent_memory(monkeypatch, capfd):
    # two rows per world for the Landmark table: the dry run is repeated after each growth.
    # The persistent arena holds exactly one pass's meshes, so a pass that did not reclaim
    # the previous one's would overflow it.
    W, steps, cfg = GOLDENS["navmesh_w9_s60"]
    _, _, _, want = load_golden("navmesh_w9_s60")
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "2")
    monkeypatch.setenv("MADRONA_B200_VERBOSE", "1")
    monkeypatch.setenv("MADRONA_B200_PERSIST_BYTES", str(_persist_need(want["mesh"][0])))
    got, _ = rollout_gpu("navmesh", W, 20, None, cfg)
    assert "grown to" in capfd.readouterr().err
    assert_traces_equal(got, {k: v[:21] for k, v in want.items()})


@pytest.mark.gpu
def test_persistent_arena_too_small_for_the_meshes(monkeypatch):
    import madrona_b200 as mb
    from sims import make_executor
    W, _, cfg = GOLDENS["navmesh_w9_s60"]
    _, _, _, want = load_golden("navmesh_w9_s60")
    monkeypatch.setenv("MADRONA_B200_PERSIST_BYTES", str(_persist_need(want["mesh"][0]) - 128))
    with pytest.raises(mb.MadronaB200Error, match="persistent arena overflow"):
        make_executor("navmesh", W, **cfg)


@pytest.mark.gpu
def test_tmp_arena_too_small_for_the_dijkstra_scratch(monkeypatch):
    import madrona_b200 as mb
    from sims import make_executor
    W, _, cfg = GOLDENS["navmesh_w9_s60"]
    _, _, _, want = load_golden("navmesh_w9_s60")
    T = want["mesh"][0][:, 1].astype(np.int64)
    r256 = lambda b: (b + 255) // 256 * 256
    plan_bytes = 4864
    init_need = int(sum(r256(plan_bytes) + r256(4 * t) + r256(8 * t) + r256(48 * t) for t in T))
    # three agents per mesh: Dijkstra (distances, entry points, heap, heap index) and BFS (queue, visited)
    agent_need = lambda t: 4 * r256(4 * t) + r256(12 * t) + r256(t)
    shared_T = int(want["mesh"][0][0, 4])
    step_need = int(sum(3 * agent_need(t) + 3 * agent_need(shared_T) for t in T))
    assert step_need > init_need + 4096
    monkeypatch.setenv("MADRONA_B200_TMP_BYTES", str(init_need + 4096))
    ex = make_executor("navmesh", W, **cfg)
    g = ex.buildLaunchGraphAllTaskGraphs()
    with pytest.raises(mb.MadronaB200Error, match="tmp allocator overflow"):
        ex.run(g)
    del g
    ex.close()


@pytest.mark.gpu
def test_bad_polygon_in_device_build_raises():
    import madrona_b200 as mb
    from sims import make_executor
    with pytest.raises(mb.MadronaB200Error, match="navmesh polygon with fewer than 3 vertices"):
        make_executor("navmesh", 4, seed=3, bad_polygon=True)
    # a good build right after
    got, _ = rollout_gpu("navmesh", 4, 2, None, {"seed": 3})
    assert (got["mesh"][0][:, 1] > 0).all()


@pytest.mark.gpu
def test_profile_names_the_navmesh_nodes():
    from sims import make_executor
    ex = make_executor("navmesh", 64, seed=3)
    prof = ex.profileNodes(reps=2)
    ex.close()
    kinds = " ".join(p["kind"] for p in prof)
    for fn in ("dijkstraSystem", "bfsSystem", "moveSystem"):
        assert fn in kinds, kinds


@pytest.mark.gpu
def test_search_node_kernels_have_no_local_memory():
    import importlib.util
    from sims import make_executor
    make_executor("navmesh", 4, seed=1).close()        # the module is compiled and cached
    spec = importlib.util.spec_from_file_location("bench_navmesh", os.path.join(ROOT, "scripts", "bench_navmesh.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    local = bench.kernel_local_bytes()
    nodes = {k: v for k, v in local.items() if "nodeKern" in k and "navmesh" in k}
    assert any("dijkstraSystem" in k for k in nodes) and any("bfsSystem" in k for k in nodes), sorted(local)
    assert all(v == 0 for v in nodes.values()), nodes
