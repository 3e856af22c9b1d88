"""Cost of the surface normal output in the batch ray caster: the render graph of `gallery` at
16384 worlds, 64 x 64 RGBD, 2 views per world, 40 props (staged instance list) and 100 props
(per-world TLAS), with normals off and on.  On, every hit pixel also reads its triangle's three
vertices and its instance's transform and writes 4 B.

The render graph is timed alone with CUDA events after a warm-up; off and on are measured in
alternating rounds.  Prints the card and its power limit with the numbers, one JSON line per
(props, normals).

    python scripts/bench_normals.py [--worlds 16384] [--res 64] [--props 40,100]
                                    [--iters 20] [--rounds 2]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench_render_aspect import _power_limit  # noqa: E402


def _time_render(worlds, props, res, normals, warmup, iters):
    import torch
    from sims import make_executor
    ex = make_executor("gallery", worlds, num_props=props, seed=7, resolution=res, rgbd=True, normals=normals)
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
    ap.add_argument("--worlds", type=int, default=16384)
    ap.add_argument("--res", type=int, default=64)
    ap.add_argument("--props", default="40,100")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()

    import torch
    card = torch.cuda.get_device_name(0)
    power = _power_limit()
    views = 2 * args.worlds
    for props in (int(p) for p in args.props.split(",")):
        times = {False: [], True: []}
        for _ in range(args.rounds):
            for normals in (False, True):
                times[normals].append(_time_render(args.worlds, props, args.res, normals, args.warmup, args.iters))
        for normals, t in times.items():
            best = min(t)
            # bytes the ray caster writes per frame: RGBA8 + f32 depth (+ int8 x 4 normal)
            written = views * args.res * args.res * (12 if normals else 8)
            print(json.dumps({
                "card": card, "power_limit": power,
                "worlds": args.worlds, "views": views, "props": props, "path": "flat" if props <= 64 else "tlas",
                "res": args.res, "normals": normals,
                "render_ms": [round(x, 4) for x in t], "best_ms": round(best, 4),
                "output_bytes_per_frame": written,
            }), flush=True)


if __name__ == "__main__":
    main()
