"""Cost of physics ray queries (mb2_trace_physics_rays / MWCudaExecutor.tracePhysicsRays):
- `room` at 8192 worlds, 16 and 256 rays per world (rays from each world's two agents in a
  fan of directions, built in torch from the exported agent positions), in world-major order
  and shuffled;
- `rays` at 1024 and 4096 bodies per world (MADRONA_B200_MAX_BODIES_PER_WORLD: the
  block-per-world kernel with the boxes in shared memory), its 64 rays per world repeated to
  256;
- beside them, the device time of room's lidar node (2 agents x 16 rays per world, traceRay
  in the simulator) from profileNodes.

Each case: --warmup calls, then one pair of CUDA events on the executor's stream around --iters
back-to-back calls, divided by --iters.  The calls go through the raw C ABI into preallocated
outputs (no tensor allocation).  Prints the card and its power limit with the numbers, one JSON
line per case.  DESIGN.md's figures come from `--iters 30`.

    python scripts/bench_physics_rays.py [--worlds 8192] [--iters 50]
"""
import argparse
import ctypes
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


def _caller(ex, world, origin, direction):
    """A closure that traces the batch into preallocated outputs through the C ABI."""
    import torch
    import madrona_b200.executor as mbe
    n = world.shape[0]
    out = (torch.empty((n, 2), dtype=torch.int32, device="cuda"), torch.empty(n, device="cuda"),
           torch.empty((n, 3), device="cuda"))
    rays = mbe._PhysicsRaysC(world.data_ptr(), origin.data_ptr(), direction.data_ptr(), None)
    hits = mbe._PhysicsRayHitsC(*[x.data_ptr() for x in out])

    def call():
        if ex._lib.mb2_trace_physics_rays(ex._h, ctypes.byref(rays), n, ctypes.byref(hits), None) != 0:
            raise RuntimeError(mbe._last_error(ex._lib))
    return call


def _case(ex, name, world, origin, direction, args, extra):
    import torch
    stream = torch.cuda.ExternalStream(ex.stream)
    ms = _timed(_caller(ex, world, origin, direction), stream, args.warmup, args.iters)
    n = int(world.shape[0])
    print(json.dumps(dict(case=name, rays=n, ms=round(ms, 4), rays_per_s=round(n / (ms * 1e-3)), **extra)),
          flush=True)


def _shuffled(world, origin, direction):
    import torch
    p = torch.randperm(world.shape[0], generator=torch.Generator().manual_seed(0)).cuda()
    return world[p].contiguous(), origin[p].contiguous(), direction[p].contiguous()


def bench_room(args, card):
    import torch
    from sims import make_executor
    W = args.worlds
    ex = make_executor("room", W, episode_len=200, seed=1)
    g = ex.buildLaunchGraphAllTaskGraphs()
    for _ in range(5):
        ex.run(g)
    pos = ex.tensor(6, "float32", (W, 2, 3)).clone()
    for per_world in (16, 256):
        fan = per_world // 2
        ang = torch.arange(fan, device="cuda", dtype=torch.float32) * (2 * torch.pi / fan)
        dirs = torch.stack([torch.cos(ang), torch.sin(ang), torch.zeros_like(ang)], dim=1)      # [fan, 3]
        origin = (pos[:, :, None, :] + torch.tensor([0, 0, 0.25], device="cuda")).expand(W, 2, fan, 3)
        origin = (origin + 0.8 * dirs).reshape(-1, 3).contiguous()
        direction = dirs.expand(W, 2, fan, 3).reshape(-1, 3).contiguous()
        world = torch.arange(W, dtype=torch.int32, device="cuda").repeat_interleave(per_world)
        extra = dict(sim="room", worlds=W, per_world=per_world, card=card[0], power_limit_w=card[1])
        _case(ex, f"room_{per_world}_world_major", world, origin, direction, args, extra)
        _case(ex, f"room_{per_world}_shuffled", *_shuffled(world, origin, direction), args, extra)
    # room's own lidar node: 2 agents x 16 rays per world, traceRay in the simulator
    try:
        prof = ex.profileNodes(reps=args.iters)
        for node in prof if isinstance(prof, list) else prof.get("nodes", []):
            if "lidar" in json.dumps(node):
                print(json.dumps(dict(case="room_lidar_node", rays=W * 32, node=node, card=card[0],
                                      power_limit_w=card[1])), flush=True)
    except Exception as e:   # profiling is an extra; the ray numbers above stand without it
        print(json.dumps(dict(case="room_lidar_node", error=str(e))), flush=True)
    del g
    ex.close()


def bench_large(args, card):
    import torch
    from sims import make_executor
    for bodies, W in ((1024, 64), (4096, 16)):
        env = {"MADRONA_B200_ROWS_PER_WORLD": str(bodies), "MADRONA_B200_PERSIST_BYTES": str(1 << 30),
               "MADRONA_B200_MAX_CANDIDATES_PER_WORLD": str(16 * bodies),
               "MADRONA_B200_MAX_CONTACTS_PER_WORLD": str(8 * bodies),
               "MADRONA_B200_MAX_BODIES_PER_WORLD": str(bodies)}
        os.environ.update(env)
        ex = make_executor("rays", W, seed=3, episode_len=0, uniform_bodies=bodies)
        g = ex.buildLaunchGraphAllTaskGraphs()
        for _ in range(3):
            ex.run(g)
        o = ex.tensor(0, "float32", (W, 64, 3)).repeat(1, 4, 1).reshape(-1, 3).contiguous()
        d = ex.tensor(1, "float32", (W, 64, 3)).repeat(1, 4, 1).reshape(-1, 3).contiguous()
        world = torch.arange(W, dtype=torch.int32, device="cuda").repeat_interleave(256)
        extra = dict(sim="rays", worlds=W, bodies=bodies, per_world=256, card=card[0], power_limit_w=card[1])
        _case(ex, f"rays_b{bodies}_world_major", world, o, d, args, extra)
        _case(ex, f"rays_b{bodies}_shuffled", *_shuffled(world, o, d), args, extra)
        del g
        ex.close()
        for k in env:
            del os.environ[k]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_physics_rays.py needs a GPU")
    card = (torch.cuda.get_device_name(0), _power_limit())
    bench_room(args, card)
    bench_large(args, card)


if __name__ == "__main__":
    main()
