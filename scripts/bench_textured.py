"""Cost of texture sampling in the batch ray caster: the render graph of `gallery`
(flat material colours) against `gallery_textured` (the same scene, two of four
materials textured, the ground wrapped), at 4096 worlds of 64 x 64 RGBD with 40
props (staged instance list) and 100 props (per-world TLAS).

The render graph is timed alone with CUDA events after a warm-up; each (props,
fixture) pair is measured in alternating rounds.  Prints the card and its power
limit with the numbers, one JSON line per configuration.

    python scripts/bench_textured.py [--worlds 4096] [--res 64] [--iters 50] [--rounds 3]
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


def _time_render(name, worlds, props, res, warmup, iters):
    import torch
    from sims import make_executor
    ex = make_executor(name, worlds, num_props=props, seed=7, resolution=res, rgbd=True)
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
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    card = torch.cuda.get_device_name(0)
    power = _power_limit()
    for props in (40, 100):
        times = {"gallery": [], "gallery_textured": []}
        for _ in range(args.rounds):
            for name in times:
                times[name].append(_time_render(name, args.worlds, props, args.res, args.warmup, args.iters))
        plain, textured = min(times["gallery"]), min(times["gallery_textured"])
        print(json.dumps({
            "card": card, "power_limit": power, "worlds": args.worlds, "resolution": args.res,
            "props": props, "path": "flat" if props <= 64 else "tlas",
            "render_ms": {k: [round(t, 4) for t in v] for k, v in times.items()},
            "best_ms": {"gallery": round(plain, 4), "gallery_textured": round(textured, 4)},
            "sampling_cost_pct": round(100.0 * (textured - plain) / plain, 2),
        }), flush=True)


if __name__ == "__main__":
    main()
