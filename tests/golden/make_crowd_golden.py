"""Generates the golden trace and reference digests of the large-world fixture sims/crowd and
its crowd2 variant (tests/test_large_physics_worlds.py) on the *reference* CPU backend, with
the harnesses that oracle/crowd.mk builds.  Run where the reference sources exist:

    make -C oracle -f crowd.mk crowd && python tests/golden/make_crowd_golden.py [name ...]

With names, only those goldens and digest cases are (re)written; the other entries of
crowd_digests.json are kept as they are.  Each digest case is run at two worker counts, and
nothing is written unless both give the same digests: the reference's broadphase queries use
fixed 32-entry stacks, and a world whose trees outgrow them would depend on the scheduling.
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

WORKER_COUNTS = (1, 4)

if __name__ == "__main__":
    names = set(sys.argv[1:])
    unknown = names - set(CROWD_GOLDENS) - set(CROWD_REFERENCE_CASES)
    if unknown:
        sys.exit(f"unknown cases: {sorted(unknown)}")
    for name, (W, steps, cfg) in sorted(CROWD_GOLDENS.items()):
        if names and name not in names:
            continue
        outs, _ = run_reference(SIMS["crowd"], W, steps, {}, cfg, workers=1)
        save_golden(name, {}, outs, W, steps)
        print(name, W, "worlds", steps, "steps")

    digests = {}
    if names and os.path.exists(CROWD_DIGESTS_PATH):
        with open(CROWD_DIGESTS_PATH) as f:
            digests = json.load(f)
    for case, (sim, W, steps, cfg) in sorted(CROWD_REFERENCE_CASES.items()):
        if names and case not in names:
            continue
        runs = [trace_digests(run_reference(SIMS[sim], W, steps, {}, cfg, workers=n)[0]) for n in WORKER_COUNTS]
        if runs[0] != runs[1]:
            differ = sorted(k for k in runs[0] if runs[0][k] != runs[1].get(k))
            sys.exit(f"{case}: columns {differ} differ between {WORKER_COUNTS} workers; nothing written")
        digests[case] = runs[0]
        print(case, sim, W, "worlds", steps, "steps")
    with open(CROWD_DIGESTS_PATH, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")
