"""Hulls past the narrowphase's staging caps (MADRONA_B200_MAX_HULL_SIZE), measured on the GPU:

(a) hullpile_big (sims/objects.py hullpile_big_specs: 24-gon prisms, a 16-gon bipyramid, an
    icosphere, an 11-gon pyramid among boxes, wedges and spheres) at 4096 worlds with the
    knob at 96 and at 255: device time per step (CUDA events around the launch graph) and,
    from a torch.profiler trace of its own, the time of physNarrowphaseLargeKernel and of
    the group-per-pair physNarrowphaseKernel per substep;
(b) room at 8192 worlds with the knob unset and at 255, alternating, three runs each: no
    primitive of room is large, so both run the same kernels;
(c) hullpile (hulls at the staging caps among balls and capped boxes) at 4096 worlds with the
    knob unset, three runs: its spheres select the sphere - hull path of physNarrowphaseKernel,
    which no bench.py workload runs.

    python scripts/bench_large_hulls.py [--steps 100] [--warmup 60]

Prints one JSON line; the card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KNOB = "MADRONA_B200_MAX_HULL_SIZE"
SUBSTEPS = 4          # sims/hullpile


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = (s.strip() for s in out.split(","))
    return name, limit


def set_knob(value):
    if value is None:
        os.environ.pop(KNOB, None)
    else:
        os.environ[KNOB] = str(value)


def timed_steps(ex, graph, steps, before_step=None):
    import torch
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for t in range(steps):
        if before_step:
            before_step(t)
        ex.run(graph)
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / steps


def kernel_ms_per_launch(ex, graph, steps, names):
    """Mean device time of the kernels whose name contains each of `names`, over `steps` steps."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            ex.run(graph)
        torch.cuda.synchronize()
    out = {}
    for name in names:
        hits = [e for e in prof.events() if name in e.name]
        total_us = sum(e.device_time_total for e in hits)
        out[name] = {"launches": len(hits), "ms": round(total_us / 1000.0 / max(len(hits), 1), 5)}
    return out


def hullpile_big(worlds, knob, steps, warmup):
    from sims import make_executor
    set_knob(knob)
    ex = make_executor("hullpile_big", worlds, seed=41)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(warmup):        # the column falls and piles up
        ex.run(graph)
    ms = timed_steps(ex, graph, steps)
    kernels = kernel_ms_per_launch(ex, graph, 20, ["physNarrowphaseLargeKernel", "physNarrowphaseKernel"])
    res = {"max_hull_size": knob, "worlds": worlds, "ms_per_step": round(ms, 4),
           "kernels_in_graph": graph.num_kernels,
           "large_kernel_ms_per_substep": kernels["physNarrowphaseLargeKernel"]["ms"],
           "large_kernel_launches_per_step": kernels["physNarrowphaseLargeKernel"]["launches"] / 20,
           "small_kernel_ms_per_substep": kernels["physNarrowphaseKernel"]["ms"]}
    assert res["large_kernel_launches_per_step"] == SUBSTEPS, res
    del graph
    ex.close()
    return res


def hullpile(worlds, steps, warmup):
    from sims import make_executor
    set_knob(None)
    ex = make_executor("hullpile", worlds, seed=41)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(warmup):        # the column falls and piles up
        ex.run(graph)
    ms = timed_steps(ex, graph, steps)
    kernel = kernel_ms_per_launch(ex, graph, 20, ["physNarrowphaseKernel"])["physNarrowphaseKernel"]
    assert kernel["launches"] == 20 * SUBSTEPS, kernel
    del graph
    ex.close()
    return round(ms, 4), kernel["ms"]


def room(worlds, knob, steps, warmup):
    import numpy as np
    import torch
    from sims import make_executor
    from trace_utils import make_inputs
    set_knob(knob)
    ex = make_executor("room", worlds, episode_len=100, seed=21)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    ins = make_inputs("room", worlds, 32, seed=9)
    actions = torch.from_numpy(np.ascontiguousarray(ins["action"])).cuda()
    act = ex.tensor(1, "int32", (worlds, 2, 3))

    def before_step(t):
        act.copy_(actions[t % 32])

    for t in range(warmup):
        before_step(t)
        ex.run(graph)
    ms = timed_steps(ex, graph, steps, before_step)
    n_kernels = graph.num_kernels
    del graph
    ex.close()
    return ms, n_kernels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=60)
    ap.add_argument("--pile-worlds", type=int, default=4096)
    ap.add_argument("--room-worlds", type=int, default=8192)
    ap.add_argument("--sphere-worlds", type=int, default=4096)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    name, limit = card()

    pile = [hullpile_big(args.pile_worlds, knob, args.steps, args.warmup) for knob in (96, 255)]

    runs = {"unset": [], "255": []}
    kernels = {}
    for _ in range(3):
        for knob in (None, 255):
            ms, n = room(args.room_worlds, knob, args.steps, args.warmup)
            key = "unset" if knob is None else str(knob)
            runs[key].append(round(ms, 4))
            kernels[key] = n
    spheres = [hullpile(args.sphere_worlds, args.steps, args.warmup) for _ in range(3)]
    set_knob(None)
    print(json.dumps({
        "gpu": name, "power_limit": limit, "steps": args.steps, "warmup": args.warmup,
        "hullpile_big": pile,
        "room": {"worlds": args.room_worlds, "ms_per_step": runs, "kernels_in_graph": kernels,
                 "mean_ms_per_step": {k: round(sum(v) / len(v), 4) for k, v in runs.items()}},
        "hullpile": {"worlds": args.sphere_worlds, "ms_per_step": [ms for ms, _ in spheres],
                     "narrowphase_ms_per_substep": [k for _, k in spheres]}}))


if __name__ == "__main__":
    main()
