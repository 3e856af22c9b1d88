"""Cost of free views (MWCudaExecutor.renderFreeViews) in the batch ray caster, on `gallery` at
4096 worlds with 40 props (staged instance list) or 100 props (per-world TLAS), RGBD:
- one 64 x 64 free view per world (each world's first camera) against the render graph's 2
  camera views per world of the same scene, per megapixel, to show whether the free path costs
  what the render graph does per pixel;
- 8 worlds at 512 x 512 (worlds 0-7's first cameras);
- one 1920 x 1080 view, with the tile chunks per view (gridDim.x) the call uses.

Every call is timed alone with CUDA events on the executor's stream after a warm-up.  Prints
the card and its power limit with the numbers, one JSON line per (props, case).

    python scripts/bench_free_views.py [--worlds 4096] [--props 40,100] [--iters 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))

from bench_render_aspect import _power_limit  # noqa: E402


def _timed(fn, stream, warmup, iters):
    import torch
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    for _ in range(iters):
        fn()
    end.record(stream)
    end.synchronize()
    return start.elapsed_time(end) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, default=4096)
    ap.add_argument("--props", default="40,100")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()

    import numpy as np
    import torch
    from sims import make_executor
    from test_raycast_free_views_model import free_grid
    card = torch.cuda.get_device_name(0)
    power = _power_limit()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    W = args.worlds
    for props in (int(p) for p in args.props.split(",")):
        ex = make_executor("gallery", W, num_props=props, seed=7, resolution=64, rgbd=True)
        step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
        ex.run(step)
        stream = torch.cuda.ExternalStream(ex.stream)
        vpos = ex.tensor(6, "float32", (W, 2, 3)).cpu().numpy()
        vrot = ex.tensor(7, "float32", (W, 2, 4)).cpu().numpy()
        views = [(w, vpos[w, 0] + np.float32([0, 0, 0.25]), vrot[w, 0], 70.0) for w in range(W)]
        rows = []
        graph_ms = _timed(lambda: ex.runAsync(render, stream), stream, args.warmup, args.iters)
        rows.append(("render_graph_64x64", 2 * W, 64, 64, graph_ms, 1))
        for name, n, w, h in [("free_64x64", W, 64, 64), ("free_512x512", 8, 512, 512),
                              ("free_1920x1080", 1, 1920, 1080)]:
            ms = _timed(lambda: ex.renderFreeViews(views[:n], w, h, rgb=True, depth=True, stream=stream),
                        stream, args.warmup, args.iters)
            rows.append((name, n, w, h, ms, free_grid(n, w, h, sms)[0]))
        ex.run(render)        # surfaces any device error of the timed frames
        for name, n, w, h, ms, chunks in rows:
            print(json.dumps({
                "card": card, "power_limit": power, "worlds": W, "props": props,
                "path": "flat" if props <= 64 else "tlas", "case": name, "views": n, "width": w, "height": h,
                "ms": round(ms, 4), "ms_per_mpixel": round(ms / (n * w * h / 1e6), 4), "chunks_per_view": chunks,
            }), flush=True)
        del step, render
        ex.close()


if __name__ == "__main__":
    main()
