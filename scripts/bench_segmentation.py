"""Cost of the segmentation output in the batch ray caster: the render graph of `gallery` at
4096 worlds, 64 x 64 RGBD, 2 views per world, 40 props (staged instance list) and 100 props
(per-world TLAS), with segmentation off and on.  On, every pixel also writes its hit entity's
id (4 B), read from the hit instance's record.

The render graph is timed alone with CUDA events after a warm-up; off and on are measured in
alternating rounds.  Prints the card and its power limit with the numbers, one JSON line per
(props, segmentation).

    python scripts/bench_segmentation.py [--worlds 4096] [--res 64] [--props 40,100]
                                         [--iters 50] [--rounds 3]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench_render_aspect import _power_limit  # noqa: E402


def _time_render(worlds, props, res, segmentation, warmup, iters):
    import torch
    from sims import make_executor
    ex = make_executor("gallery", worlds, num_props=props, seed=7, resolution=res, rgbd=True,
                       segmentation=segmentation)
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
    ap.add_argument("--res", type=int, default=64)
    ap.add_argument("--props", default="40,100")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    card = torch.cuda.get_device_name(0)
    power = _power_limit()
    views = 2 * args.worlds
    for props in (int(p) for p in args.props.split(",")):
        times = {False: [], True: []}
        for _ in range(args.rounds):
            for seg in (False, True):
                times[seg].append(_time_render(args.worlds, props, args.res, seg, args.warmup, args.iters))
        for seg, t in times.items():
            best = min(t)
            # bytes the ray caster writes per frame: RGBA8 + f32 depth (+ i32 entity id)
            written = views * args.res * args.res * (12 if seg else 8)
            print(json.dumps({
                "card": card, "power_limit": power,
                "worlds": args.worlds, "views": views, "props": props, "path": "flat" if props <= 64 else "tlas",
                "res": args.res, "segmentation": seg,
                "render_ms": [round(x, 4) for x in t], "best_ms": round(best, 4),
                "output_bytes_per_frame": written,
            }), flush=True)


if __name__ == "__main__":
    main()
