"""Generates tests/golden/render_digests.json: SHA-256 of the RGB and depth images the
batch ray caster writes for room_render and the gallery at 40 and 100 props (worlds of up
to 128 instances, the warp-built TLAS and the staged instance list).  The stored digests
were made by the engine before instance lists became compact and large worlds got their
own TLAS builder; tests/test_render_large_worlds.py checks the output is still identical.
Needs an H100:

    python tests/golden/make_render_digests.py
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
DIGESTS_PATH = os.path.join(ROOT, "tests", "golden", "render_digests.json")

CASES = {
    # name: (sim, worlds, steps, cfg, rgb slot, depth slot, views per world)
    "room_render": ("room_render", 4, 5, {"episode_len": 20, "seed": 3, "resolution": 32, "rgbd": True}, 13, 14, 2),
    "gallery_40": ("gallery", 3, 3, {"num_props": 40, "seed": 5, "resolution": 40, "rgbd": True}, 8, 9, 2),
    "gallery_100": ("gallery", 3, 3, {"num_props": 100, "seed": 5, "resolution": 40, "rgbd": True}, 8, 9, 2),
}


def render_digests():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from sims import make_executor
    out = {}
    for name, (sim, W, steps, cfg, rgb_slot, depth_slot, views) in CASES.items():
        ex = make_executor(sim, W, **cfg)
        step, render = ex.buildLaunchGraphAllTaskGraphs(), ex.buildRenderGraph()
        for _ in range(steps):
            ex.run(step)
        ex.run(render)
        res = cfg["resolution"]
        rgb = ex.tensor(rgb_slot, "uint8", (views * W, res, res, 4)).cpu().numpy()
        depth = ex.tensor(depth_slot, "float32", (views * W, res, res)).cpu().numpy()
        ex.close()
        out[name] = {"rgb": hashlib.sha256(rgb.tobytes()).hexdigest(),
                     "depth": hashlib.sha256(depth.tobytes()).hexdigest()}
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else DIGESTS_PATH
    with open(path, "w") as f:
        json.dump(render_digests(), f, indent=1, sort_keys=True)
        f.write("\n")
