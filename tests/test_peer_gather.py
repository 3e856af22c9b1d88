"""NVLink peer-store gather (include/madrona_b200.h mb2_peer_gather_*) on one GPU: a single-rank
loop-back, and 2 to 16 ranks in one process, one executor per rank, connected by
mb2_peer_gather_connect_local.  Every rank's gathered columns are compared bit for bit with the
ranks' exported columns and with one executor of all the worlds.  The IPC path between
processes is exercised by `bench.py --gpus N`; the host-side sharding logic by
tests/test_sharding.py with gloo; the store plan and flag protocol by
tests/test_peer_gather_model.py."""
import numpy as np
import pytest


@pytest.mark.gpu
def test_loopback_gather_matches_exported_columns():
    import torch
    from sims import SIMS, make_executor
    from trace_utils import make_inputs

    W, steps = 257, 9
    ex = make_executor("cartpole", W, max_steps=50, seed=4)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    desc = SIMS["cartpole"]
    outs = [s for s in desc.outputs]
    pg = ex.peerGather([s.slot for s in outs], [(W,) + s.per_world for s in outs], [s.dtype for s in outs], 1, 0)
    pg.connect([pg.local_handle()])
    ins = make_inputs("cartpole", W, steps, seed=2)
    act = ex.tensor(1, "int32", (W, 1))
    stream = torch.cuda.current_stream()
    cols = [ex.tensor(s.slot, s.dtype, (W,) + s.per_world) for s in outs]
    for t in range(steps):
        act.copy_(torch.from_numpy(np.ascontiguousarray(ins["action"][t])))
        ex.runAsync(graph, stream)
        pg.push(stream)
        pg.wait(stream)
        torch.cuda.synchronize()
        for i, c in enumerate(cols):
            got = pg.tensor(t & 1, i)
            assert got.shape == c.shape and torch.equal(got, c), (t, outs[i].name)
        pg.release(stream)
    pg.close()
    ex.close()


def _bits(t):
    """A tensor's bytes, so that equality is bit for bit (NaNs and signed zeros included)."""
    import torch
    return t.contiguous().reshape(-1).view(torch.uint8)


def _gathered_slots(sim):
    from sims import SIMS
    fixed = [s for s in SIMS[sim].outputs if not s.dynamic]
    if sim == "room":
        # all 7 fixed outputs plus the reward again: kMaxGatherSlots slots of 20 B to 256 B per world
        fixed.append(fixed[0])
    return fixed


def _run_ranks(sim, W, N, steps, cfg, input_seed):
    """N executors of W worlds (rank r: worlds [r W, (r + 1) W)) and one of N W worlds, stepped
    on one stream in bench.py's order: every rank's run(k) and push(k), then every rank's
    wait(k - 1), read and release(k - 1).  Checks every rank's gathered columns of every step."""
    import torch
    import madrona_b200 as mb
    from madrona_b200 import sharding
    from sims import SIMS, make_executor
    from trace_utils import make_inputs

    desc = SIMS[sim]
    base = int(cfg.pop("seed"))
    slots = _gathered_slots(sim)
    exs = [make_executor(sim, W, seed=sharding.world_seed(base, r * W, 0), **cfg) for r in range(N)]
    whole = make_executor(sim, N * W, seed=base, **cfg)
    graphs = [ex.buildLaunchGraphAllTaskGraphs() for ex in exs]
    whole_graph = whole.buildLaunchGraphAllTaskGraphs()
    pgs = [ex.peerGather([s.slot for s in slots], [(W,) + s.per_world for s in slots],
                         [s.dtype for s in slots], N, r) for r, ex in enumerate(exs)]
    mb.PeerGather.connect_local(pgs)

    ins = make_inputs(sim, N * W, steps, seed=input_seed)
    if "reset" in ins:
        # no respawns: a respawned entity's ID comes from a pool shared by the executor's worlds
        ins["reset"][:] = 0
    in_t = [{s.name: ex.tensor(s.slot, s.dtype, (W,) + s.per_world) for s in desc.inputs} for ex in exs]
    whole_in = {s.name: whole.tensor(s.slot, s.dtype, (N * W,) + s.per_world) for s in desc.inputs}
    cols = [[ex.tensor(s.slot, s.dtype, (W,) + s.per_world) for s in slots] for ex in exs]
    whole_cols = [whole.tensor(s.slot, s.dtype, (N * W,) + s.per_world) for s in slots]
    stream = torch.cuda.current_stream()
    want = {}

    def consume(k):
        got = []
        for pg in pgs:
            pg.wait(stream)
            got.append([pg.tensor(k & 1, i).clone() for i in range(len(slots))])
            pg.release(stream)
        exported, reference = want.pop(k)
        for i, s in enumerate(slots):
            assert torch.equal(_bits(exported[i]), _bits(reference[i])), \
                f"step {k} {s.name}: {N} ranks of {W} worlds differ from one executor of {N * W}"
            for r in range(N):
                assert torch.equal(_bits(got[r][i]), _bits(exported[i])), \
                    f"step {k} {s.name}: rank {r}'s gathered column differs from the exported columns"

    for k in range(steps):
        step_in = {name: torch.from_numpy(np.ascontiguousarray(v[k])).cuda() for name, v in ins.items()}
        exported = []
        for r in range(N):
            for name, t in in_t[r].items():
                t.copy_(sharding.local_slice(step_in[name], r, N))
            exs[r].runAsync(graphs[r], stream)
            exported.append([c.clone() for c in cols[r]])
            pgs[r].push(stream)
        for name, t in whole_in.items():
            t.copy_(step_in[name])
        whole.runAsync(whole_graph, stream)
        want[k] = ([torch.cat([e[i] for e in exported]) for i in range(len(slots))],
                   [c.clone() for c in whole_cols])
        if k >= 1:
            consume(k - 1)
    consume(steps - 1)
    torch.cuda.synchronize()
    for pg in pgs:
        pg.close()
    for ex in exs + [whole]:
        ex.close()


# (sim, worlds per rank, ranks, sim cfg).  Cartpole's state / reward / done slices of 257 worlds
# are 4112 / 1028 / 1028 B, so the ranks' slices start at every residue mod 16; 16 ranks of 3
# worlds have 12 B reward and done slices (tail words only).  The room's 1023 worlds make a
# 261888 B lidar slice (more than one grid-stride pass of the push grid) and an 8184 B reward
# slice, so rank 1 starts 8 B off a 16-byte boundary.
RANK_CASES = [
    ("cartpole", 257, 2, {"max_steps": 200, "seed": 40}),
    ("cartpole", 257, 3, {"max_steps": 200, "seed": 41}),
    ("cartpole", 257, 4, {"max_steps": 200, "seed": 42}),
    ("cartpole", 257, 8, {"max_steps": 200, "seed": 43}),
    ("cartpole", 3, 16, {"max_steps": 200, "seed": 44}),
    ("room", 5, 2, {"episode_len": 100, "seed": 45}),
    ("room", 5, 4, {"episode_len": 100, "seed": 46}),
    ("room", 1023, 2, {"episode_len": 100, "seed": 47}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("sim,W,N,cfg", RANK_CASES, ids=[f"{c[0]}-w{c[1]}-n{c[2]}" for c in RANK_CASES])
def test_ranks_of_one_process_gather_every_step_bit_exact(sim, W, N, cfg, monkeypatch):
    if N > 8:
        # 17 executors on a shared device: a tmp arena far below the 256 MiB default is plenty
        monkeypatch.setenv("MADRONA_B200_TMP_BYTES", str(16 << 20))
    _run_ranks(sim, W, N, steps=12, cfg=dict(cfg), input_seed=N * 1000 + W)


@pytest.mark.gpu
def test_rejected_gather_calls_name_the_problem_and_change_nothing():
    import torch
    import madrona_b200 as mb
    from sims import SIMS, make_executor

    W = 4
    slots = SIMS["cartpole"].outputs
    spec = ([s.slot for s in slots], [(W,) + s.per_world for s in slots], [s.dtype for s in slots])
    exs = [make_executor("cartpole", W, seed=100 + r * W) for r in range(2)]
    graphs = [ex.buildLaunchGraphAllTaskGraphs() for ex in exs]
    ex = exs[0]

    def refused(match, fn, *args):
        with pytest.raises(mb.MadronaB200Error, match=match):
            fn(*args)

    refused(r"num_slots must be 1 to 8, got 0", ex.peerGather, [], [], [], 1, 0)
    refused(r"num_slots must be 1 to 8, got 9", ex.peerGather, [3] * 9, [(W,)] * 9, ["float32"] * 9, 1, 0)
    refused(r"world_size must be 1 to 16, got 0", ex.peerGather, *spec, 0, 0)
    refused(r"world_size must be 1 to 16, got 17", ex.peerGather, *spec, 17, 0)
    refused(r"rank 2 is not below world_size 2", ex.peerGather, *spec, 2, 2)
    refused(r"entry 1: 3 bytes per rank is not a multiple of 4", ex.peerGather,
            [2, 3], [(W, 4), (3,)], ["float32", "uint8"], 1, 0)
    refused(r"export slot 7 \(entry 0\) is not in use", ex.peerGather, [7], [(W,)], ["int32"], 1, 0)

    g = [e.peerGather(*spec, 2, r) for r, e in enumerate(exs)]
    fewer_slots = exs[1].peerGather(spec[0][:2], spec[1][:2], spec[2][:2], 2, 1)
    other_bytes = exs[1].peerGather(spec[0], [(W - 1,) + s.per_world for s in slots], spec[2], 2, 1)
    closed = exs[1].peerGather(*spec, 2, 1)
    closed.close()
    refused(r"gathers\[1\] is null", mb.PeerGather.connect_local, [g[0], closed])
    refused(r"no gathers", mb.PeerGather.connect_local, [])
    refused(r"gathers\[0\] has world_size 2, but 1 gathers were given", mb.PeerGather.connect_local, [g[0]])
    refused(r"rank 0 appears twice", mb.PeerGather.connect_local, [g[0], g[0]])
    refused(r"gathers\[0\] is rank 1", mb.PeerGather.connect_local, [g[1], g[0]])
    refused(r"gathers\[1\] has 2 slots, gathers\[0\] 3", mb.PeerGather.connect_local, [g[0], fewer_slots])
    refused(r"gathers\[1\] slot 0 has 48 bytes per rank, gathers\[0\] 64", mb.PeerGather.connect_local,
            [g[0], other_bytes])
    if torch.cuda.device_count() >= 2:
        far = make_executor("cartpole", W, gpu_id=1, seed=104)
        far_gather = far.peerGather(*spec, 2, 1)
        refused(r"gathers\[1\] is on GPU 1, gathers\[0\] on GPU 0", mb.PeerGather.connect_local,
                [g[0], far_gather])
        far_gather.close()
        far.close()
    torch.cuda.synchronize()

    # nothing was launched or connected: both executors run, and the gathers connect and gather
    mb.PeerGather.connect_local(g)
    stream = torch.cuda.current_stream()
    cols = [[e.tensor(s.slot, s.dtype, (W,) + s.per_world) for s in slots] for e in exs]
    exported = {}

    def consume(k):
        for r in range(2):
            g[r].wait(stream)
            for i in range(len(slots)):
                want = torch.cat([e[i] for e in exported[k]])
                assert torch.equal(_bits(g[r].tensor(k & 1, i)), _bits(want)), (k, r, slots[i].name)
            g[r].release(stream)

    for k in range(3):
        exported[k] = []
        for r in range(2):
            exs[r].runAsync(graphs[r], stream)
            exported[k].append([c.clone() for c in cols[r]])
            g[r].push(stream)
        if k >= 1:
            consume(k - 1)
    consume(2)
    torch.cuda.synchronize()
    for pg in g + [fewer_slots, other_bytes]:
        pg.close()
    for e in exs:
        e.close()
