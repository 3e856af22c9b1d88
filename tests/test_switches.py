"""Code paths kept behind switches for A/B measurements must stay correct: each runs the
parity tests of the kernels it touches in a child process (the switches are read once per
process).

  MADRONA_B200_SORT_FUSE_COPYBACK=1   copy-back of exported columns as work items of the
                                      rearrange kernel (default: separate launch, DESIGN 3.1)
  MADRONA_B200_PDL=1                  programmatic dependent launch of every engine kernel:
                                      each must reach pdlSync() before it touches memory
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = {
    "fused_copy_back": ({"MADRONA_B200_SORT_FUSE_COPYBACK": "1"},
                        ["tests/test_sort_sweep.py", "tests/test_sort_custom_key.py", "tests/test_gridworld.py"],
                        None),
    "pdl": ({"MADRONA_B200_PDL": "1"},
            ["tests/test_sort_sweep.py", "tests/test_sort_custom_key.py", "tests/test_gridworld.py",
             "tests/test_room.py"], None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_parity_holds_with_switch(case):
    env, targets, select = CASES[case]
    cmd = [sys.executable, "-m", "pytest", *targets, "-m", "gpu", "-q", "-x", "--tb=short", "-p", "no:cacheprovider"]
    if select:
        cmd += ["-k", select]
    res = subprocess.run(cmd, cwd=ROOT, env={**os.environ, **env}, capture_output=True, text=True, timeout=900)
    tail = (res.stdout + res.stderr)[-3000:]
    assert res.returncode == 0, tail      # 0 = every selected test passed
    assert " passed" in res.stdout, tail    # ... and something was selected
