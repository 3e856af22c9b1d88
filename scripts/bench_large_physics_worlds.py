"""Worlds of more than 128 bodies (MADRONA_B200_MAX_BODIES_PER_WORLD), measured on the GPU:

(a) crowd (sims/crowd) with 64, 256, 1024 and 4096 bodies in every world, the world count
    scaled to about a million bodies, the knob at 4096: device time per step (CUDA events
    around the launch graph, no episode reset in the window) and, from torch.profiler traces
    of their own, the time per launch of the warp-per-world and block-per-world candidate
    searches, the narrowphase, both solves, and of the rebuild on the step that builds every
    world's tree (the first one);
(b) bench.py's flagship (room, 8192 worlds) with the knob unset and at 4096, three
    alternating runs each of `bench.py --gpus 1 --steps 200 --warmup 20`.

    python scripts/bench_large_physics_worlds.py [--steps 100] [--warmup 20] [--bodies 1048576] [--sizes 64,256,1024,4096] [--skip-room]

Prints one JSON line; the card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KNOB = "MADRONA_B200_MAX_BODIES_PER_WORLD"
KERNELS = ["physFindCandidatesKernel", "physFindCandidatesLargeKernel", "physNarrowphaseKernel",
           "physSolvePositionsKernel", "physSolveVelocitiesKernel"]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = (s.strip() for s in out.split(","))
    return name, limit


def crowd_env(bodies):
    """Room for `bodies` per world: rows, the BVHs in the persistent arena, pairs."""
    os.environ[KNOB] = "4096"
    os.environ["MADRONA_B200_ROWS_PER_WORLD"] = str(bodies + 64)
    os.environ["MADRONA_B200_PERSIST_BYTES"] = str(3 << 30)
    os.environ["MADRONA_B200_MAX_CANDIDATES_PER_WORLD"] = str(max(16 * bodies, 1024))
    os.environ["MADRONA_B200_MAX_CONTACTS_PER_WORLD"] = str(max(8 * bodies, 512))


def timed_steps(ex, graph, steps):
    import torch
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(steps):
        ex.run(graph)
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps


def profiled(ex, graph, steps, names):
    """Per name: launches and mean / max device ms per launch over `steps` steps."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            ex.run(graph)
        torch.cuda.synchronize()
    out = {}
    for name in names:
        hits = [e.device_time_total for e in prof.events() if name in e.name and e.device_time_total > 0]
        out[name] = {"launches": len(hits), "ms": round(sum(hits) / 1000.0 / max(len(hits), 1), 5),
                     "max_ms": round(max(hits, default=0) / 1000.0, 5)}
    return out


def crowd(bodies, worlds, steps, warmup):
    from sims import make_executor
    crowd_env(bodies)
    ex = make_executor("crowd", worlds, seed=7, episode_len=0, uniform_bodies=bodies)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    # the first step rebuilds every world's tree (the constructor reset the broadphase)
    rebuild = profiled(ex, graph, 1, ["physRebuildKernel"])["physRebuildKernel"]
    for _ in range(warmup):
        ex.run(graph)
    ms = timed_steps(ex, graph, steps)
    kernels = profiled(ex, graph, 10, KERNELS)
    res = {"bodies_per_world": bodies, "worlds": worlds, "ms_per_step": round(ms, 4),
           "kernels_in_graph": graph.num_kernels,
           "rebuild_ms_on_reset_step": rebuild["max_ms"],
           "kernel_ms_per_launch": {k: v["ms"] for k, v in kernels.items()},
           "launches_per_step": {k: v["launches"] / 10 for k, v in kernels.items()}}
    del graph
    ex.close()
    return res


def bench_py(knob, steps, warmup):
    env = dict(os.environ)
    for k in ("MADRONA_B200_ROWS_PER_WORLD", "MADRONA_B200_PERSIST_BYTES",
              "MADRONA_B200_MAX_CANDIDATES_PER_WORLD", "MADRONA_B200_MAX_CONTACTS_PER_WORLD", KNOB):
        env.pop(k, None)
    if knob is not None:
        env[KNOB] = str(knob)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps),
                          "--warmup", str(warmup)], capture_output=True, text=True, env=env, cwd=ROOT)
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    if out.returncode != 0 or not lines:
        raise RuntimeError(out.stderr[-2000:])
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--bodies", type=int, default=1 << 20, help="bodies per crowd run, all worlds together")
    ap.add_argument("--sizes", default="64,256,1024,4096")
    ap.add_argument("--bench-steps", type=int, default=200)
    ap.add_argument("--bench-warmup", type=int, default=20)
    ap.add_argument("--skip-room", action="store_true")
    ap.add_argument("--room-runs", type=int, default=3, help="bench.py runs per knob setting, alternating")
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    name, limit = card()

    results = {"gpu": name, "power_limit": limit, "steps": args.steps, "warmup": args.warmup, "crowd": []}
    for n in (int(s) for s in args.sizes.split(",") if s):
        results["crowd"].append(crowd(n, max(1, args.bodies // n), args.steps, args.warmup))
        print(json.dumps(results["crowd"][-1]), file=sys.stderr, flush=True)

    if not args.skip_room:
        runs = {"unset": [], "4096": []}
        for _ in range(args.room_runs):
            for knob in (None, 4096):
                r = bench_py(knob, args.bench_steps, args.bench_warmup)
                runs["unset" if knob is None else "4096"].append(r)
                print(json.dumps({"knob": knob, "bench_py": r}), file=sys.stderr, flush=True)
        results["room_bench_py"] = runs
    print(json.dumps(results))


if __name__ == "__main__":
    main()
