"""Generates tests/golden/*.npz by running the fixture simulators on the
*reference* CPU backend (oracle/_ref, built from the reference sources by
oracle/Makefile), and tests/golden/reference_digests.json from the larger
roll-outs of trace_utils.REFERENCE_CASES.  Run where the reference sources exist:

    make -C oracle && python tests/golden/make_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.runner import run_reference  # noqa: E402
from sims import SIMS  # noqa: E402
from trace_utils import (DIGESTS_PATH, REFERENCE_CASES, make_inputs, reference_case,  # noqa: E402
                         reference_columns, save_golden, trace_digests)

CASES = [
    # (file, sim, worlds, steps, cfg)
    ("cartpole_w64_s300", "cartpole", 64, 300, {"max_steps": 200, "seed": 0}),
    ("cartpole_w3_s50", "cartpole", 3, 50, {"max_steps": 10, "seed": 7}),
    ("gridworld_w32_s150", "gridworld", 32, 150,
     {"grid_size": 6, "episode_len": 40, "init_items": 6, "seed": 11}),
    # tiny grid + long episodes: many pickups, item table saturates at kMaxItems
    ("gridworld_w5_s400", "gridworld", 5, 400,
     {"grid_size": 3, "episode_len": 97, "init_items": 20, "seed": 3}),
    # rigid-body room: two resets inside the trace (episode_len 100 + random resets)
    ("room_w4_s210", "room", 4, 210, {"episode_len": 100, "seed": 21}),
    # same fixture with agent 0 grabbing / releasing cubes through fixed joints
    ("room_grab_w3_s120", "room", 3, 120, {"episode_len": 70, "seed": 5, "grab_period": 5}),
    # Hide&Seek-class arena: wedge / hexagonal hulls, latched doors (fixed joints to static
    # walls), grab (fixed) and shove (one-step hinge) joints, two resets inside the trace
    ("arena_w2_s200", "arena", 2, 200, {"episode_len": 90, "seed": 17}),
    # Solver::TGS through the same API (tgs.cpp: integrate velocities / positions only)
    ("room_tgs_w3_s45", "room_tgs", 3, 45, {"episode_len": 30, "seed": 8}),
    # spheres: sphere-sphere, sphere-plane and sphere-hull (GJK) contacts
    ("balls_w6_s160", "balls", 6, 160, {"seed": 3}),
    # 95 bodies per world: candidate search beyond one 64-leaf mask word, ~300 contacts per world
    ("balls_many_w2_s60", "balls_many", 2, 60, {"seed": 9}),
    # hulls at the narrowphase's staging caps, compound bodies, spheres inside hulls
    ("hullpile_w4_s150", "hullpile", 4, 150, {"seed": 41}),
    # 60 bodies per world: hull contacts on bodies the position solve does not stage
    ("hullpile_many_w2_s100", "hullpile_many", 2, 100, {"seed": 43}),
]

if __name__ == "__main__":
    only = sys.argv[1:]
    for name, sim, W, steps, cfg in CASES:
        if only and name not in only:
            continue
        inputs = make_inputs(sim, W, steps, seed=1234)
        outs, _ = run_reference(SIMS[sim], W, steps, inputs, cfg, workers=1)
        save_golden(name, inputs, outs, W, steps)
        print(name, {k: (v.shape if not isinstance(v, list) else f"{len(v)} frames")
                     for k, v in outs.items()})

    # per-column digests of the reference traces of trace_utils.REFERENCE_CASES (all of
    # them; or, named on the command line, only those, merged into the existing file)
    named = [name for name in only if name in REFERENCE_CASES]
    if not only or "reference_digests" in only or named:
        import json
        digests = {}
        if named and "reference_digests" not in only:
            with open(DIGESTS_PATH) as f:
                digests = json.load(f)
        for name in (named or REFERENCE_CASES):
            sim, W, steps, inputs, cfg = reference_case(name)
            outs, _ = run_reference(SIMS[sim], W, steps, inputs, cfg, workers=4)
            digests[name] = trace_digests(reference_columns(name, outs))
            print(name, W, "worlds", steps, "steps")
        with open(DIGESTS_PATH, "w") as f:
            json.dump(digests, f, indent=1, sort_keys=True)
            f.write("\n")

    # digest of the reference GJK probe (oracle/gjk_probe.cpp built against the
    # reference's src/physics/gjk.hpp + geo.cpp): lets the engine's header be
    # checked where oracle/_ref/gjk_probe_ref is absent
    if not only or "gjk_probe" in only:
        import hashlib
        import subprocess
        probe = os.path.join(ROOT, "oracle", "_ref", "gjk_probe_ref")
        text = subprocess.run([probe], capture_output=True, text=True, check=True).stdout
        with open(os.path.join(ROOT, "tests", "golden", "gjk_probe.sha256"), "w") as f:
            f.write(hashlib.sha256(text.encode()).hexdigest() + "\n")
        print("gjk_probe", len(text.splitlines()), "values")
