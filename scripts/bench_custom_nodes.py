"""The same per-row work as a ParallelForNode and as an addDynamicCountNode, on the
customnodes_bench build of sims/customnodes at gridworld-like sizes (65536 worlds, about
10 Token rows per world): device time of each node (CUDA events, mb2_profile_nodes), of
the dynamic-count node's one-thread count node, and of the count latch.  The latch is
timed on the probe build with a dynamic count of 0, where the run node is the latch
kernel plus a launch whose blocks exit at once.

    python scripts/bench_custom_nodes.py [--worlds 65536] [--steps 100] [--warmup 10]

Prints one JSON line; the card name and power limit are read in the same run."""
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


def node_ms(prof, prefix):
    hits = [p for p in prof if p["kind"].startswith(prefix)]
    assert len(hits) == 1, (prefix, [p["kind"] for p in prof])
    return round(hits[0]["ms"], 5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    import torch
    from sims import make_executor

    assert torch.cuda.is_available(), "needs a GPU"
    name, limit = card()
    W = args.worlds

    ex = make_executor("customnodes_bench", W, seed=1)
    graph = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(args.warmup):
        ex.run(graph)
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.steps):
        ex.run(graph)
    stop.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(stop) / args.steps
    rows = ex.exportedNumRows(5)
    prof = ex.profileNodes(reps=args.steps)
    del graph
    ex.close()

    probe = make_executor("customnodes_probe", 1, count=0, threads=1, dynamic=0)
    latch_prof = probe.profileNodes(reps=args.steps)
    probe.close()

    print(json.dumps({
        "workload": "customnodes_bench", "worlds": W, "token_rows": rows, "steps": args.steps,
        "ms_per_step": round(ms, 4), "gpu": name, "power_limit": limit,
        "parallel_for_ms": node_ms(prof, "parallel_for:"),
        "dynamic_count_run_ms": node_ms(prof, "custom:customnodes::TokenRowsNode::run"),
        "dynamic_count_count_ms": node_ms(prof, "custom:madrona::TaskGraphBuilder::dynamicCountWrapper<customnodes::TokenRowsNode>"),
        "latch_plus_empty_run_ms": node_ms(latch_prof, "custom:customnodes::ProbeNode::run"),
        "nodes": prof}))


if __name__ == "__main__":
    main()
