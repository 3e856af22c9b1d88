"""Custom task-graph nodes: TaskGraphBuilder::addNodeFn, addOneOffNode, addDynamicCountNode
and node data, on sims/customnodes.  The reference CPU backend runs the same fixture with
its per-world addNodeFn form; its trace is kept as a golden (customnodes_w23_s40.npz) and
as per-column digests of a larger roll-out (custom_nodes_digests.json), both written by
tests/golden/make_custom_nodes_golden.py.  The probe build of the fixture
(customnodes_probe) records every run of a node with a fixed count N and T threads per
invocation."""
import glob
import json
import os
import re

import numpy as np
import pytest

from trace_utils import GOLDEN_DIR, assert_traces_equal, load_golden, rollout_gpu, trace_digests

# golden -> (worlds, steps, sim cfg); worlds 3, 10 and 17 never have tokens
GOLDENS = {"customnodes_w23_s40": (23, 40, {"seed": 7})}
# case -> (worlds, steps, sim cfg)
DIGEST_CASES = {"customnodes_w300_s60": (300, 60, {"seed": 4100})}
DIGESTS_PATH = os.path.join(GOLDEN_DIR, "custom_nodes_digests.json")
# most resident 256-thread blocks an H100 can hold: 132 SMs x 2048 threads
H100_MAX_RESIDENT_BLOCKS = 132 * 2048 // 256
PROBE_SLOTS = 4096
# (node type, mangled function) of every custom node function in the fixture
CUSTOM_NODE_FNS = [(n, "3runEi") for n in ("SpawnNode", "WarpSumNode", "TokenRowsNode", "SetCountNode",
                                          "CoopNode", "CensusNode")] + [("TokenRowsNode", "dynamicCountWrapper")]


def _digests():
    with open(DIGESTS_PATH) as f:
        return json.load(f)


# ---- CPU: the goldens exercise the feature -------------------------------------------------

def test_golden_exercises_dynamic_counts_and_churn():
    W, steps, _, outs = load_golden("customnodes_w23_s40")
    rows = np.array([len(f) for f in outs["token_out"]])
    # the dynamic-count node's count (live Token rows) varies, and drops to 0 on whole steps
    assert len(np.unique(rows[1:])) > 10 and (rows[1:] == 0).sum() >= 3
    # CoopNode's latched count varies and is 0 on some steps
    k = outs["coop"][1:, :, 0]
    assert (k == k[:, :1]).all() and set(np.unique(k)) >= {0, 1, 3, 6}
    # the warp-per-world reduction counts what the table holds; empty worlds stay empty
    counts = outs["world_sum"][1:, :, 0]
    assert (counts.sum(axis=1) == rows[1:]).all()
    assert (counts[:, [3, 10, 17]] == 0).all() and (counts.max(axis=0)[[0, 1, 2]] > 0).all()
    # the second task graph runs once per step; entity IDs are recycled
    assert (outs["census"][:, :, 0] == np.arange(steps + 1)[:, None]).all()
    made = outs["census"][-1, :, 2]
    ids = np.concatenate([f[:, 1] for f in outs["token_entity"]])
    assert len(np.unique(ids)) < made.sum()
    # every live token's hash was written this step
    assert all((f != 0).all() for f in outs["token_out"][1:])


def test_digest_case_count_exceeds_the_persistent_grid():
    counts = _digests()["customnodes_w300_s60"]["coop_counts"]
    assert min(counts) == 0 and max(counts) > H100_MAX_RESIDENT_BLOCKS


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_reference_reproduces_golden(name):
    from oracle import runner
    from sims import SIMS
    W, steps, cfg = GOLDENS[name]
    if not runner.available("customnodes"):
        pytest.skip("needs oracle/_ref/ref_customnodes (make -C oracle -f customnodes.mk customnodes)")
    _, _, _, want = load_golden(name)
    got, _ = runner.run_reference(SIMS["customnodes"], W, steps, None, cfg, workers=1)
    assert_traces_equal(got, want)


def test_fixture_jit_compiles_a_kernel_per_custom_node(tmp_path, monkeypatch):
    import madrona_b200 as mb
    from sims import SIMS
    desc = SIMS["customnodes"]
    monkeypatch.setenv("MADRONA_B200_KERNEL_CACHE_DIR", str(tmp_path))
    monkeypatch.delenv("MADRONA_B200_NO_KERNEL_CACHE", raising=False)
    mb.precompile(mb.CompileConfig(userSources=desc.sources,
                                   userCompileFlags=["-I" + os.path.dirname(desc.sources[0])]))
    (cubin,) = glob.glob(str(tmp_path / "*.cubin"))
    data = open(cubin, "rb").read()
    kerns = set(re.findall(rb"_ZN7madrona5mwGPU8nodeKernINS0_6FnNodeI[0-9A-Za-z_]+", data))
    metas = set(re.findall(rb"_ZN7madrona5mwGPU8nodeMetaINS0_6FnNodeI[0-9A-Za-z_]+", data))
    for node, fn in CUSTOM_NODE_FNS:
        tag = f"{len(node)}{node}E".encode()
        assert any(tag in k and fn.encode() in k for k in kerns), f"no nodeKern for {node} {fn}"
        assert any(tag in m and fn.encode() in m for m in metas), f"no nodeMeta for {node} {fn}"


# ---- GPU: parity ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_matches_golden(name):
    W, steps, cfg = GOLDENS[name]
    _, _, _, want = load_golden(name)
    got, n_kernels = rollout_gpu("customnodes", W, steps, None, cfg)
    assert n_kernels > 0
    assert sorted(got) == sorted(want)
    assert_traces_equal(got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(DIGEST_CASES))
def test_matches_reference_digests(case):
    W, steps, cfg = DIGEST_CASES[case]
    got, _ = rollout_gpu("customnodes", W, steps, None, cfg)
    want = _digests()[case]["digests"]
    have = trace_digests(got)
    assert sorted(have) == sorted(want)
    assert [k for k in sorted(want) if have[k] != want[k]] == []


@pytest.mark.gpu
def test_matches_live_reference():
    from oracle import runner
    from sims import SIMS
    if not runner.available("customnodes"):
        pytest.skip("needs oracle/_ref/ref_customnodes")
    W, steps, cfg = 61, 45, {"seed": 99}
    want, _ = runner.run_reference(SIMS["customnodes"], W, steps, None, cfg, workers=2)
    got, _ = rollout_gpu("customnodes", W, steps, None, cfg)
    assert_traces_equal(got, want)


@pytest.mark.gpu
def test_parallel_branches_and_profile_names():
    from sims import make_executor
    ex = make_executor("customnodes", 64, seed=3)
    g = ex.buildLaunchGraph([0])
    assert g.num_branches >= 3
    del g
    prof = ex.profileNodes(reps=2)
    kinds = [p["kind"] for p in prof]
    ex.close()
    for want in ["custom:customnodes::SpawnNode::run", "custom:customnodes::WarpSumNode::run",
                 "custom:customnodes::TokenRowsNode::run", "custom:customnodes::SetCountNode::run",
                 "custom:customnodes::CoopNode::run", "custom:customnodes::CensusNode::run"]:
        assert want in kinds, kinds
    assert any(k.startswith("custom:") and "dynamicCountWrapper" in k for k in kinds), kinds


# ---- GPU: invocation probe -----------------------------------------------------------------

def _run_probe(count, threads, dynamic=0, extra_node_datas=0):
    from sims import make_executor
    ex = make_executor("customnodes_probe", 1, count=count, threads=threads, dynamic=dynamic,
                       extra_node_datas=extra_node_datas)
    try:
        g = ex.buildLaunchGraphAllTaskGraphs()
        ex.run(g)
        n = ex.exportedNumRows(6)
        rows = ex.tensor(6, "uint32", (n, 14)).cpu().numpy().copy()
        info = ex.tensor(7, "uint32", (1, 2)).cpu().numpy().copy()
        del g
    finally:
        ex.close()
    return rows, info


def _check_probe(rows, info, N, T):
    assert rows.shape == (PROBE_SLOTS, 14)
    u64 = lambda lo, hi: rows[:, lo].astype(np.uint64) | (rows[:, hi].astype(np.uint64) << np.uint64(32))
    s = np.arange(PROBE_SLOTS, dtype=np.uint64)
    n_s = np.where(s < N % PROBE_SLOTS, N // PROBE_SLOTS + 1, N // PROBE_SLOTS).astype(np.uint64)
    # invocations i < N with i % slots == s: s, s + slots, ...
    idx_sum = n_s * s + np.uint64(PROBE_SLOTS) * (n_s * (n_s - np.uint64(1)) // np.uint64(2))
    idx_sum[n_s == 0] = 0
    T64 = np.uint64(T)
    assert (rows[:, 0].astype(np.uint64) == T64 * n_s).all(), "an invocation ran a wrong number of times"
    assert (u64(2, 3) == T64 * idx_sum).all(), "the invocations that ran are not 0 .. N-1"
    assert (u64(4, 5) == n_s * np.uint64(T * (T - 1) // 2)).all(), "lanes ran an invocation unevenly"
    full = np.zeros(8, dtype=np.uint32)
    full[:T // 32] = 0xFFFFFFFF
    if T < 32:
        full[0] = (1 << T) - 1
    lanes = rows[:, 6:14]
    assert (lanes[n_s > 0] == full).all(), "not every lane threadIdx % T ran"
    assert (lanes[n_s == 0] == 0).all()
    assert int(info[0, 0]) == N, "an invocation at or above N ran"


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 2, 32, 64, 256])
@pytest.mark.parametrize("N", [0, 1, 255, 256, 257, 1_000_003])
def test_probe_fixed_count(N, T):
    rows, info = _run_probe(N, T)
    _check_probe(rows, info, N, T)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 256])
@pytest.mark.parametrize("N", [0, 257, 1_000_003])
def test_probe_node_that_zeroes_its_count_runs_the_latched_count(N, T):
    rows, info = _run_probe(N, T, dynamic=1)
    _check_probe(rows, info, N, T)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [0, 3, 512])
def test_bad_threads_per_invocation_fails_creation(T):
    import madrona_b200 as mb
    with pytest.raises(mb.MadronaB200Error, match="num_threads_per_invocation"):
        _run_probe(5, T)
    rows, info = _run_probe(300, 32)
    _check_probe(rows, info, 300, 32)


@pytest.mark.gpu
def test_too_many_node_datas_fails_creation():
    import madrona_b200 as mb
    with pytest.raises(mb.MadronaB200Error, match="too many custom node datas"):
        _run_probe(5, 1, extra_node_datas=1100)
    # right at the limit (the probe node's own data is the 1024th)
    rows, info = _run_probe(5, 1, extra_node_datas=1023)
    _check_probe(rows, info, 5, 1)
