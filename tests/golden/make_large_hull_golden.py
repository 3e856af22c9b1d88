"""Generates the golden traces and reference digests of the large-hull fixtures
(tests/test_large_hulls.py: the hullpile simulators with hulls past the narrowphase's staging
caps) on the *reference* CPU backend, with the hullpile harness binaries oracle/Makefile
builds.  Run where the reference sources exist:

    make -C oracle && python tests/golden/make_large_hull_golden.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.runner import run_reference  # noqa: E402
from trace_utils import save_golden, trace_digests  # noqa: E402
from test_large_hulls import (GOLDENS, LARGE_DIGESTS_PATH, LARGE_REFERENCE_CASES,  # noqa: E402
                              reference_desc)

if __name__ == "__main__":
    for name, (sim, W, steps, cfg) in sorted(GOLDENS.items()):
        outs, _ = run_reference(reference_desc(sim), W, steps, {}, cfg, workers=1)
        save_golden(name, {}, outs, W, steps)
        print(name, W, "worlds", steps, "steps")

    digests = {}
    for case, (sim, W, steps, cfg) in sorted(LARGE_REFERENCE_CASES.items()):
        outs, _ = run_reference(reference_desc(sim), W, steps, {}, cfg, workers=4)
        digests[case] = trace_digests(outs)
        print(case, W, "worlds", steps, "steps")
    with open(LARGE_DIGESTS_PATH, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")
