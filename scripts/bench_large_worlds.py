"""Ray casting large worlds: `gallery_sized` at 1024 worlds x {512, 2048, 8192} props per
world (every 17th hidden, so a little fewer instances), 64 x 64 RGBD, two views per world.
All three sizes go through the global-memory TLAS builder (worlds above 128 instances) and
the TLAS traversal.

Per size: the render-prepare node (instance gather + TLAS build) from mb2_profile_nodes,
and the render graph alone timed with CUDA events after a warm-up.  Prints the card and
its power limit with the numbers, one JSON line per size.

    python scripts/bench_large_worlds.py [--worlds 1024] [--props 512,2048,8192] [--res 64]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _measure(worlds, props, res, warmup, iters, reps):
    import torch
    from sims import make_executor
    # room for every prop from the start: no table growth inside the timed window
    os.environ["MADRONA_B200_ROWS_PER_WORLD"] = str(props + 256)
    ex = make_executor("gallery_sized", worlds, props=[props] * worlds, seed=7, resolution=res, rgbd=True)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    for _ in range(3):
        ex.run(step)
    nodes = ex.profileNodes(reps=reps)
    prepare = [n for n in nodes if n["kind"] == "render_prepare"]
    stream = torch.cuda.ExternalStream(ex.stream)
    for _ in range(warmup):
        ex.runAsync(render, stream)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    for _ in range(iters):
        ex.runAsync(render, stream)
    end.record(stream)
    end.synchronize()
    ex.run(render)        # surfaces any device error of the timed frames
    render_ms = start.elapsed_time(end) / iters
    step_ms = sum(n["ms"] for n in nodes)
    del step, render
    ex.close()
    return (prepare[0]["ms"] if prepare else None), step_ms, render_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, default=1024)
    ap.add_argument("--props", default="512,2048,8192")
    ap.add_argument("--res", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import torch
    card = torch.cuda.get_device_name(0)
    power = _power_limit()
    for props in [int(p) for p in args.props.split(",")]:
        visible = props - (props - 1) // 17
        prepare_ms, step_ms, render_ms = _measure(args.worlds, props, args.res, args.warmup, args.iters, args.reps)
        # the TLAS build reads each instance record (80 B) and writes at most one 60 B node
        # per instance; the sort and tree passes touch 8 B keys and 52 B scratch entries
        print(json.dumps({
            "card": card, "power_limit": power, "worlds": args.worlds, "resolution": args.res,
            "props": props, "instances_per_world": visible,
            "render_prepare_ms": None if prepare_ms is None else round(prepare_ms, 4),
            "step_nodes_ms": round(step_ms, 4),
            "render_graph_ms": round(render_ms, 4),
        }), flush=True)


if __name__ == "__main__":
    main()
