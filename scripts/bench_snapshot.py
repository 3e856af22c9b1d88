"""Executor snapshots at training sizes: room at 8192 worlds and arena at 4096.  For each,
the snapshot buffer's size (every table and arena at its capacity), the bytes a save
copies (the live part), the device time of one save and one restore (CUDA events around
each launch on the executor's stream, median of --reps), one step's time beside them, and
2 x copied bytes / time against the H100 SXM's 3.35 TB/s of HBM3.

    python scripts/bench_snapshot.py [--reps 20] [--warmup 5]

Prints one JSON line; the card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_GBPS = 3350.0


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = (s.strip() for s in out.split(","))
    return name, limit


def measure(sim, W, cfg, reps, warmup):
    import numpy as np
    import torch
    from sims import SIMS, make_executor
    from trace_utils import make_inputs

    ex = make_executor(sim, W, **cfg)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    desc = SIMS[sim]
    ins = make_inputs(sim, W, 1, seed=3)
    for s in desc.inputs:
        ex.tensor(s.slot, s.dtype, (W,) + s.per_world).copy_(torch.from_numpy(np.ascontiguousarray(ins[s.name][0])))
    torch.cuda.synchronize()
    for _ in range(warmup):
        ex.run(graph)
    stream = torch.cuda.ExternalStream(ex.stream)

    def timed(fn):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(reps):
            start.record(stream)
            fn()
            stop.record(stream)
            stop.synchronize()
            times.append(start.elapsed_time(stop))
        return float(np.median(times))

    snap = ex.snapshot()
    snap.save()
    for _ in range(warmup):
        snap.save()
        snap.restore()
    save_ms = timed(snap.save)
    restore_ms = timed(snap.restore)
    step_ms = timed(lambda: ex.runAsync(graph, ex.stream))
    snap.save()
    nbytes, copied = snap.nbytes, snap.saved_nbytes
    snap.close()
    del graph
    ex.close()

    def gbps(ms):
        return round(2 * copied / (ms * 1e-3) / 1e9, 1)
    return {"workload": sim, "worlds": W, "snapshot_bytes": nbytes, "copied_bytes": copied,
            "save_ms": round(save_ms, 4), "restore_ms": round(restore_ms, 4), "step_ms": round(step_ms, 4),
            "save_gbps": gbps(save_ms), "restore_gbps": gbps(restore_ms), "hbm_gbps": HBM_GBPS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    name, limit = card()
    results = [measure("room", 8192, {"episode_len": 100, "seed": 1}, args.reps, args.warmup),
               measure("arena", 4096, {"episode_len": 100, "seed": 1}, args.reps, args.warmup)]
    print(json.dumps({"bench": "snapshot", "gpu": name, "power_limit": limit, "results": results}))


if __name__ == "__main__":
    main()
