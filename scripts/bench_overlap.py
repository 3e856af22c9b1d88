"""Device time of the overlap-query fixtures at 8192 worlds -- sims/triggers (broadphase +
standalone overlap rows + user queries, no solver) and sims/buttons (XPBD step, then
findEntitiesWithinAABB per button and checkEntityAABBOverlap per agent) -- plus the
per-node breakdown (candidate search, overlap-row node, the user query nodes).

    python scripts/bench_overlap.py [--worlds 8192] [--steps 200] [--warmup 20]

Prints one JSON line per fixture; the card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = (s.strip() for s in out.split(","))
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()

    import numpy as np
    import torch
    from sims import make_executor
    from sims.inputs import buttons_inputs, triggers_inputs

    assert torch.cuda.is_available(), "needs a GPU"
    name, limit = card()
    W = args.worlds
    fixtures = [
        ("triggers", {"seed": 1}, triggers_inputs),
        ("buttons", {"episode_len": 200, "seed": 1}, buttons_inputs),
    ]
    for sim, cfg, make_inputs in fixtures:
        ex = make_executor(sim, W, **cfg)
        graph = ex.buildLaunchGraphAllTaskGraphs()
        act = ex.tensor(1 if sim == "buttons" else 0, "int32", (W, 2, 3 if sim == "buttons" else 2))
        ins = make_inputs(W, args.warmup + args.steps, seed=3)["action"]
        for t in range(args.warmup):
            act.copy_(torch.from_numpy(np.ascontiguousarray(ins[t])))
            ex.run(graph)
        # actions stay fixed inside the timed window: only the step graph is on the clock
        act.copy_(torch.from_numpy(np.ascontiguousarray(ins[args.warmup])))
        torch.cuda.synchronize()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.steps):
            ex.run(graph)
        stop.record()
        torch.cuda.synchronize()
        ms = start.elapsed_time(stop) / args.steps
        prof = ex.profileNodes(reps=20)
        ex.close()
        print(json.dumps({"workload": sim, "worlds": W, "steps": args.steps,
                          "ms_per_step": round(ms, 4), "env_steps_per_s": round(W / ms * 1e3),
                          "gpu": name, "power_limit": limit, "nodes": prof}))


if __name__ == "__main__":
    main()
