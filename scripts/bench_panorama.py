"""Cost of panoramic views in the batch ray caster: the render graph of `room_render` at 16384
worlds x 2 views, RGBD, for
  - a 64 x 64 pinhole (the flagship observation),
  - a 256 x 16 panorama (the same pixel count, 360 degrees around),
  - a 360 x 1 panorama (a 2D laser scan, one beam per degree),
  - a 1024 x 32 panorama (a 32-beam spinning lidar at 1024 columns).

The render graph is timed alone with CUDA events after a warm-up, the configurations in
alternating rounds.  Prints the card and its power limit with the numbers, one JSON line per
configuration.

    python scripts/bench_panorama.py [--worlds 16384] [--iters 30] [--rounds 3]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from bench_render_aspect import _power_limit  # noqa: E402

# (name, width, height, panorama)
CONFIGS = [
    ("pinhole_64x64", 64, 64, False),
    ("panorama_256x16", 256, 16, True),
    ("panorama_360x1", 360, 1, True),
    ("panorama_1024x32", 1024, 32, True),
]


def _time_render(worlds, width, height, panorama, warmup, iters):
    import torch
    from sims import make_executor
    size = dict(resolution=width) if width == height else dict(width=width, height=height)
    ex = make_executor("room_render", worlds, episode_len=200, seed=0, rgbd=True, panorama=panorama, **size)
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
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    card = torch.cuda.get_device_name(0)
    power = _power_limit()
    views = 2 * args.worlds
    times = {name: [] for name, _, _, _ in CONFIGS}
    for _ in range(args.rounds):
        for name, width, height, panorama in CONFIGS:
            times[name].append(_time_render(args.worlds, width, height, panorama, args.warmup, args.iters))
    for name, width, height, panorama in CONFIGS:
        t = times[name]
        best = min(t)
        rays = views * width * height
        print(json.dumps({
            "card": card, "power_limit": power, "config": name,
            "worlds": args.worlds, "views": views, "width": width, "height": height, "panorama": panorama,
            "render_ms": [round(x, 4) for x in t], "best_ms": round(best, 4),
            "primary_rays_per_s": round(rays / (best * 1e-3)),
        }), flush=True)


if __name__ == "__main__":
    main()
