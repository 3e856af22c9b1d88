"""Cost of non-square images in the batch ray caster: the render graph of `gallery` at 4096
worlds, RGBD, 2 views per world, 40 props (staged instance list) and 100 props (per-world TLAS),
at image shapes of equal pixel count: 64 x 64, 128 x 32, 32 x 128 and 4096 x 1.  The last one
runs on 32 x 1 warp tiles; to see what they buy, run it again under a build of the library
that keeps 8 x 4 tiles for every image (MADRONA_B200_LIB, as scripts/ab_bench.sh does).

The render graph is timed alone with CUDA events after a warm-up; the shapes are measured in
alternating rounds.  Prints the card and its power limit with the numbers, one JSON line per
(props, shape).

    python scripts/bench_render_aspect.py [--worlds 4096] [--shapes 64x64,128x32,32x128,4096x1]
                                          [--props 40,100] [--iters 50] [--rounds 3]
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


def _time_render(worlds, props, width, height, warmup, iters):
    import torch
    from sims import make_executor
    ex = make_executor("gallery", worlds, num_props=props, seed=7, width=width, height=height, rgbd=True)
    step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
    ex.run(step)
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
    ms = start.elapsed_time(end) / iters
    del step, render
    ex.close()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, default=4096)
    ap.add_argument("--shapes", default="64x64,128x32,32x128,4096x1")
    ap.add_argument("--props", default="40,100")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    shapes = [tuple(int(x) for x in s.split("x")) for s in args.shapes.split(",")]

    import torch
    import madrona_b200 as mb
    card = torch.cuda.get_device_name(0)
    power = _power_limit()
    views = 2 * args.worlds
    for props in (int(p) for p in args.props.split(",")):
        times = {s: [] for s in shapes}
        for _ in range(args.rounds):
            for s in shapes:
                times[s].append(_time_render(args.worlds, props, s[0], s[1], args.warmup, args.iters))
        for (w, h), t in times.items():
            best = min(t)
            print(json.dumps({
                "card": card, "power_limit": power, "library": mb.library_path(),
                "worlds": args.worlds, "views": views, "props": props, "path": "flat" if props <= 64 else "tlas",
                "width": w, "height": h,
                "render_ms": [round(x, 4) for x in t], "best_ms": round(best, 4),
                "rays_per_s": round(views * w * h / (best * 1e-3), 1),
            }), flush=True)


if __name__ == "__main__":
    main()
