"""Generates the golden trace and reference digests of the custom-node fixture
(sims/customnodes) on the *reference* CPU backend, with the harness oracle/customnodes.mk
builds (oracle/harness_customnodes.cpp).  Run where the reference sources exist:

    make -C oracle && make -C oracle -f customnodes.mk customnodes && python tests/golden/make_custom_nodes_golden.py
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
from test_custom_nodes import DIGEST_CASES, DIGESTS_PATH, GOLDENS  # noqa: E402

if __name__ == "__main__":
    for name, (W, steps, cfg) in sorted(GOLDENS.items()):
        outs, _ = run_reference(SIMS["customnodes"], W, steps, None, cfg, workers=1)
        save_golden(name, {}, outs, W, steps)
        print(name, W, "worlds", steps, "steps")

    cases = {}
    for case, (W, steps, cfg) in sorted(DIGEST_CASES.items()):
        outs, _ = run_reference(SIMS["customnodes"], W, steps, None, cfg, workers=4)
        # CoopNode's count of every step: k blocks per world, all worlds
        counts = [int(k) * W for k in outs["coop"][1:, :, 0].max(axis=1)]
        cases[case] = {"digests": trace_digests(outs), "coop_counts": counts}
        print(case, W, "worlds", steps, "steps")
    with open(DIGESTS_PATH, "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
        f.write("\n")
