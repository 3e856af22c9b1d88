"""Generates the golden trace and reference digests of the large-world fixture sims/crowd
(tests/test_large_physics_worlds.py) on the *reference* CPU backend, with the harness that
oracle/crowd.mk builds.  Run where the reference sources exist:

    make -C oracle -f crowd.mk crowd && python tests/golden/make_crowd_golden.py
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
from test_large_physics_worlds import CROWD_DIGESTS_PATH, CROWD_GOLDENS, CROWD_REFERENCE_CASES  # noqa: E402

if __name__ == "__main__":
    for name, (W, steps, cfg) in sorted(CROWD_GOLDENS.items()):
        outs, _ = run_reference(SIMS["crowd"], W, steps, {}, cfg, workers=1)
        save_golden(name, {}, outs, W, steps)
        print(name, W, "worlds", steps, "steps")

    digests = {}
    for case, (W, steps, cfg) in sorted(CROWD_REFERENCE_CASES.items()):
        outs, _ = run_reference(SIMS["crowd"], W, steps, {}, cfg, workers=1)
        digests[case] = trace_digests(outs)
        print(case, W, "worlds", steps, "steps")
    with open(CROWD_DIGESTS_PATH, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")
