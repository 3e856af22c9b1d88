"""Writes the golden trace and reference digests of the navmesh fixture (sims/navmesh) on the
*reference* CPU backend, with the harness oracle/navmesh.mk builds (oracle/harness_navmesh.cpp).
Run where the reference sources exist:

    make -C oracle && make -C oracle -f navmesh.mk navmesh && python tests/golden/make_navmesh_golden.py
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
from test_navmesh import DIGEST_CASES, DIGESTS_PATH, GOLDENS  # noqa: E402

if __name__ == "__main__":
    for name, (W, steps, cfg) in sorted(GOLDENS.items()):
        outs, _ = run_reference(SIMS["navmesh"], W, steps, None, cfg, workers=1)
        save_golden(name, {}, outs, W, steps)
        print(name, W, "worlds", steps, "steps")

    cases = {}
    for case, (W, steps, cfg) in sorted(DIGEST_CASES.items()):
        outs, _ = run_reference(SIMS["navmesh"], W, steps, None, cfg, workers=8)
        cases[case] = trace_digests(outs)
        print(case, W, "worlds", steps, "steps")
    with open(DIGESTS_PATH, "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
        f.write("\n")
