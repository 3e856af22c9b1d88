"""Generates the golden traces and reference digests of the overlap-query fixtures
(sims/triggers, sims/buttons) on the *reference* CPU backend, with the harnesses
oracle/overlap.mk builds (oracle/harness_triggers.cpp, oracle/harness_buttons.cpp).
Run where the reference sources exist:

    make -C oracle && make -C oracle -f overlap.mk overlap && python tests/golden/make_overlap_golden.py
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
from test_overlap_queries import (GOLDENS, INPUTS, OVERLAP_DIGESTS_PATH,  # noqa: E402
                                  OVERLAP_REFERENCE_CASES, overlap_case)

if __name__ == "__main__":
    for name, (sim, W, steps, cfg) in sorted(GOLDENS.items()):
        ins = INPUTS[sim](W, steps, seed=1234)
        outs, _ = run_reference(SIMS[sim], W, steps, ins, cfg, workers=1)
        save_golden(name, ins, outs, W, steps)
        print(name, W, "worlds", steps, "steps")

    digests = {}
    for case in sorted(OVERLAP_REFERENCE_CASES):
        sim, W, steps, ins, cfg = overlap_case(case)
        outs, _ = run_reference(SIMS[sim], W, steps, ins, cfg, workers=4)
        digests[case] = trace_digests(outs)
        print(case, W, "worlds", steps, "steps")
    with open(OVERLAP_DIGESTS_PATH, "w") as f:
        json.dump(digests, f, indent=1, sort_keys=True)
        f.write("\n")
