"""Navigation meshes on sims/navmesh at 8192 worlds (6 agents each, about 60-70 triangles per
mesh): executor creation time with and without the per-world meshes (each world builds its
own with Navmesh::initFromPolygons in its constructor, in every init pass), device time per
step and per node (CUDA events, mb2_profile_nodes) for the Dijkstra, BFS and movement nodes,
and each JIT'd kernel's local memory (CU_FUNC_ATTRIBUTE_LOCAL_SIZE_BYTES).

    python scripts/bench_navmesh.py [--worlds 8192] [--steps 100] [--warmup 10]

Prints a table and one JSON line; the card name and power limit are read in the same run."""
import argparse
import ctypes
import glob
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CU_FUNC_ATTRIBUTE_LOCAL_SIZE_BYTES = 3


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, limit = (s.strip() for s in out.split(","))
    return name, limit


def kernel_local_bytes(tag=b"N7navmesh"):
    """{kernel: local bytes} of the cached simulator module whose symbols contain `tag`."""
    import torch
    torch.zeros(1, device="cuda")          # a current context for the driver calls
    cache = os.environ.get("MADRONA_B200_KERNEL_CACHE_DIR") or os.path.join(ROOT, "madrona_b200", "_jit_cache")
    cu = ctypes.CDLL("libcuda.so.1")
    out = {}
    for path in glob.glob(os.path.join(cache, "*.cubin")):
        data = open(path, "rb").read()
        if tag not in data:
            continue
        mod = ctypes.c_void_p()
        assert cu.cuModuleLoadData(ctypes.byref(mod), data) == 0
        n = ctypes.c_uint()
        assert cu.cuModuleGetFunctionCount(ctypes.byref(n), mod) == 0
        fns = (ctypes.c_void_p * n.value)()
        assert cu.cuModuleEnumerateFunctions(fns, n, mod) == 0
        for f in fns:
            name, local = ctypes.c_char_p(), ctypes.c_int()
            assert cu.cuFuncGetName(ctypes.byref(name), ctypes.c_void_p(f)) == 0
            assert cu.cuFuncGetAttribute(ctypes.byref(local), CU_FUNC_ATTRIBUTE_LOCAL_SIZE_BYTES,
                                         ctypes.c_void_p(f)) == 0
            out[name.value.decode()] = local.value
        cu.cuModuleUnload(mod)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, default=8192)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()

    import torch
    from sims import make_executor

    assert torch.cuda.is_available(), "needs a GPU"
    name, limit = card()
    W = args.worlds
    res = {"workload": "navmesh", "worlds": W, "steps": args.steps, "gpu": name, "power_limit": limit}

    # an executor first, so that neither timed creation pays for loading the module
    make_executor("navmesh", 64, seed=1).close()
    for per_world in (False, True):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ex = make_executor("navmesh", W, seed=1, episode_len=50, per_world=per_world)
        torch.cuda.synchronize()
        create_ms = (time.perf_counter() - t0) * 1e3
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
        del graph
        prof = ex.profileNodes(reps=args.steps)
        ex.close()
        key = "per_world" if per_world else "shared_only"
        res[key] = {"create_ms": round(create_ms, 1), "ms_per_step": round(start.elapsed_time(stop) / args.steps, 4)}
        for node in ("dijkstraSystem", "bfsSystem", "moveSystem"):
            hits = [p["ms"] for p in prof if node in p["kind"]]
            res[key][node + "_ms"] = round(hits[0], 4) if len(hits) == 1 else None
        res[key]["nodes"] = prof

    res["local_bytes"] = kernel_local_bytes()
    print(f"{name}, power limit {limit}, {W} worlds")
    print(f"{'':14}{'create ms':>11}{'step ms':>10}{'dijkstra':>10}{'bfs':>9}{'move':>9}")
    for key in ("shared_only", "per_world"):
        r = res[key]
        print(f"{key:14}{r['create_ms']:>11}{r['ms_per_step']:>10}{r['dijkstraSystem_ms']:>10}"
              f"{r['bfsSystem_ms']:>9}{r['moveSystem_ms']:>9}")
    for k, v in sorted(res["local_bytes"].items()):
        print(f"local {v:6d} B  {k[:110]}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
