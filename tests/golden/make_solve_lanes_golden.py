"""Generates the reference digests of tests/test_velocity_solve_lanes.py: for each of its cases, a
7-world run of the *reference* CPU backend seeded S0, kept as one SHA-256 per world and exported
column (entity handles left out).  Run where the reference sources exist:

    make -C oracle && make -C oracle -f crowd.mk crowd && python tests/golden/make_solve_lanes_golden.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_velocity_solve_lanes import CASES, DIGESTS_PATH, REF_WORLDS, S0, reference_world_digests  # noqa: E402

if __name__ == "__main__":
    digests = {}
    for case in sorted(CASES):
        digests[case], _ = reference_world_digests(case)
        print(case, REF_WORLDS, "worlds from seed", S0, CASES[case][1], "steps")
    with open(DIGESTS_PATH, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")
