"""Seeded synthetic action streams of the overlap-query fixtures (sims/triggers,
sims/buttons), shared by their tests and scripts/bench_overlap.py."""
from __future__ import annotations

import numpy as np


def triggers_inputs(num_worlds: int, num_steps: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    # each choice held for 4 steps, so agents cross the pen
    act = rng.integers(0, 3, size=(num_steps // 4 + 1, num_worlds, 2, 2), dtype=np.int32)
    return {"action": np.repeat(act, 4, axis=0)[:num_steps]}


def buttons_inputs(num_worlds: int, num_steps: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    # each choice held for 6 steps: agents walk onto a button, stay a while, walk off
    n = num_steps // 6 + 1
    amount = np.where(rng.random((n, num_worlds, 2)) < 0.6, 3, rng.integers(0, 4, size=(n, num_worlds, 2)))
    angle = rng.integers(0, 8, size=(n, num_worlds, 2))
    act = np.stack([amount, angle, np.full_like(amount, 2)], axis=-1)
    act = np.repeat(act, 6, axis=0)[:num_steps].astype(np.int32)
    return {"reset": (rng.random((num_steps, num_worlds, 1)) < 0.004).astype(np.int32),
            "action": act}
