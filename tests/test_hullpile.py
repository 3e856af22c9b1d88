"""Hull fixture at the narrowphase's staging caps (sims/hullpile: an 8-gon prism dropped
onto an 8-gon pedestal, 8-gon prisms on the floor, a 16-face bipyramid, tetrahedra,
pentagonal pyramids, wedges, boxes, spheres and two compound bodies in a walled pen), GPU
engine vs the reference CPU backend.  Same bar as tests/test_balls.py: every exported
column BIT-EXACT (1e-4 only with MADRONA_B200_FAST_MATH=1).  What the goldens exercise
is checked by tests/test_hull_contact_model.py."""
import os

import numpy as np
import pytest

from oracle import runner
from sims import SIMS
from trace_utils import assert_matches_reference, assert_traces_equal, load_golden, reference_case, rollout_gpu

EXACT = os.environ.get("MADRONA_B200_FAST_MATH", "0") != "1"
CFG = {"seed": 41}
# more pairs than the defaults allow for (256 candidates, 128 contacts per world)
MANY_ENV = {"MADRONA_B200_MAX_CANDIDATES_PER_WORLD": "4096", "MADRONA_B200_MAX_CONTACTS_PER_WORLD": "2048",
            "MADRONA_B200_ROWS_PER_WORLD": "128"}
MANY_CFG = {"seed": 43}


@pytest.mark.parametrize("golden", ["hullpile_w4_s150", "hullpile_many_w2_s100"])
def test_golden_is_finite_and_above_the_floor(golden):
    W, steps, ins, outs = load_golden(golden)
    for k in ("body_pos", "body_rot", "body_vel"):
        assert np.isfinite(outs[k]).all(), k
    pos = outs["body_pos"]
    # body 0 is the plane; every other body keeps its centre above it and inside the pen
    assert pos[:, :, 1:, 2].min() > 0.05
    assert np.abs(pos[:, :, :, :2]).max() <= 6.25


@pytest.mark.skipif(not runner.available("hullpile"), reason="oracle/_ref not built")
def test_reference_backend_reproduces_golden():
    W, steps, ins, outs = load_golden("hullpile_w4_s150")
    got, _ = runner.run_reference(SIMS["hullpile"], W, steps, ins, CFG, workers=1)
    assert_traces_equal(got, outs)


@pytest.mark.skipif(not runner.available("hullpile_many"), reason="oracle/_ref not built")
def test_many_reference_backend_reproduces_golden():
    W, steps, ins, outs = load_golden("hullpile_many_w2_s100")
    got, _ = runner.run_reference(SIMS["hullpile_many"], W, steps, ins, MANY_CFG, workers=1)
    assert_traces_equal(got, outs)


@pytest.mark.gpu
def test_gpu_matches_golden():
    W, steps, ins, outs = load_golden("hullpile_w4_s150")
    got, n_kernels = rollout_gpu("hullpile", W, steps, ins, CFG)
    assert n_kernels > 10
    assert_traces_equal(got, outs, exact=EXACT, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_gpu_matches_live_reference_many_worlds():
    sim, W, steps, ins, cfg = reference_case("hullpile_w300_s120")
    got, _ = rollout_gpu(sim, W, steps, ins, cfg)
    assert_matches_reference("hullpile_w300_s120", got, exact=EXACT)


@pytest.mark.gpu
def test_many_gpu_matches_golden(monkeypatch):
    for k, v in MANY_ENV.items():
        monkeypatch.setenv(k, v)
    W, steps, ins, outs = load_golden("hullpile_many_w2_s100")
    assert outs["body_pos"].shape[2] == 60
    got, _ = rollout_gpu("hullpile_many", W, steps, ins, MANY_CFG)
    assert_traces_equal(got, outs, exact=EXACT, rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
def test_many_gpu_matches_live_reference(monkeypatch):
    for k, v in MANY_ENV.items():
        monkeypatch.setenv(k, v)
    sim, W, steps, ins, cfg = reference_case("hullpile_many_w48_s100")
    got, _ = rollout_gpu(sim, W, steps, ins, cfg)
    assert_matches_reference("hullpile_many_w48_s100", got, exact=EXACT)


@pytest.mark.gpu
def test_4096_worlds_prefix_equals_reference():
    # worlds are independent and seeded by their index: worlds [0, 64) of a 4096-world run
    # (the narrowphase's persistent grid full of hull - hull items) equal a 64-world
    # reference run bit for bit
    from test_full_size import _rollout_prefix
    sim, keep, steps, ins, cfg = reference_case("hullpile_w64_s60")
    got = _rollout_prefix(sim, 4096, steps, ins, cfg, keep)
    del got["body_entity"]           # handles come from one pool for all worlds
    assert_matches_reference("hullpile_w64_s60", got, exact=EXACT)
