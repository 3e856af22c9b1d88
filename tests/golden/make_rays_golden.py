"""Generates the reference digests and the one-world golden trace of the physics ray fixture
sims/rays (tests/test_physics_rays.py) on the *reference* CPU backend, with the harness that
oracle/rays.mk builds.  Run where the reference sources exist:

    make -C oracle -f rays.mk rays && python tests/golden/make_rays_golden.py

Each case is run at two worker counts, and nothing is written unless both give the same
digests.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.runner import run_reference  # noqa: E402
from sims import SIMS  # noqa: E402
from trace_utils import save_golden, trace_digests  # noqa: E402
from test_physics_rays import RAYS_DIGESTS_PATH, RAYS_GOLDEN, RAYS_REFERENCE_CASES  # noqa: E402

WORKER_COUNTS = (1, 4)

if __name__ == "__main__":
    digests = {}
    for case, (W, steps, cfg, _) in sorted(RAYS_REFERENCE_CASES.items()):
        runs = [run_reference(SIMS["rays"], W, steps, {}, cfg, workers=n)[0] for n in WORKER_COUNTS]
        d = [trace_digests(r) for r in runs]
        if d[0] != d[1]:
            differ = sorted(k for k in d[0] if d[0][k] != d[1].get(k))
            sys.exit(f"{case}: columns {differ} differ between {WORKER_COUNTS} workers; nothing written")
        digests[case] = d[0]
        if case == RAYS_GOLDEN:
            save_golden(case, {}, runs[0], W, steps)
        print(case, W, "worlds", steps, "steps")
    with open(RAYS_DIGESTS_PATH, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")
