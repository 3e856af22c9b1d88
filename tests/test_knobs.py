"""The MADRONA_B200_* environment variables that configure an executor are read and checked
once, before any CUDA call: unset means the default, and a set value that is malformed or out
of range fails mb2_executor_create (and mb2_jit_precompile) with the variable's name in
mb2_last_error().  Needs no GPU: with a valid value, creation of a one-world executor with an
empty simulator fails at a later step (the first CUDA call without a GPU, the simulator's
missing entry points with one), and that error names no knob."""
import ctypes

import pytest

import madrona_b200 as mb
from madrona_b200.executor import _CompileConfigC, _StateConfigC

I32_MAX = 2**31 - 1
U64_MAX = 2**64 - 1

# integer knobs: (lowest, highest) accepted value
RANGES = {
    "ROWS_PER_WORLD": (1, I32_MAX),
    "TMP_BYTES": (1, U64_MAX),
    "PERSIST_BYTES": (1, U64_MAX),
    "MAX_CANDIDATES_PER_WORLD": (1, I32_MAX),
    "MAX_CONTACTS_PER_WORLD": (1, I32_MAX),
    "MAX_HULL_SIZE": (16, 255),
    "MAX_BODIES_PER_WORLD": (128, 4096),
}
BOOLEANS = ["TABLE_GROWTH", "GRAPH_BRANCHES", "FAST_MATH", "NO_KERNEL_CACHE", "RENDER_DEBUG"]
PATHS = ["KERNEL_CACHE_DIR"]
ALL = list(RANGES) + BOOLEANS + PATHS

# values the rest of the suite sets, which must stay accepted
SUITE_VALUES = {
    "ROWS_PER_WORLD": ["2", "36", "3072"],
    "MAX_CANDIDATES_PER_WORLD": ["3", "16384"],
    "MAX_CONTACTS_PER_WORLD": ["4", "8192"],
    "PERSIST_BYTES": ["3456", str(3 << 30)],   # small: the navmesh tests set one just short of a mesh
}

MALFORMED = ["", "abc", "12x", "-1", "99999999999999999999999"]

BAD = [(k, v) for k in RANGES for v in MALFORMED + [str(RANGES[k][0] - 1), str(RANGES[k][1] + 1)]]
BAD += [(k, v) for k in BOOLEANS for v in MALFORMED + ["2", "yes", "on"]]
BAD += [(k, "") for k in PATHS]

GOOD = [(k, None) for k in ALL]   # unset: the default
GOOD += [(k, str(v)) for k in RANGES for v in RANGES[k]]
GOOD += [(k, v) for k, vs in SUITE_VALUES.items() for v in vs]
GOOD += [(k, v) for k in BOOLEANS for v in ["0", "1"]]


@pytest.fixture(scope="module")
def cache_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("knob_cache"))


@pytest.fixture
def knob_env(monkeypatch, cache_dir):
    """Clears every knob; with a GPU the empty simulator is compiled once, into cache_dir."""
    for k in ALL:
        monkeypatch.delenv("MADRONA_B200_" + k, raising=False)
    monkeypatch.setenv("MADRONA_B200_KERNEL_CACHE_DIR", cache_dir)
    return monkeypatch


def _create():
    lib = mb.load_library()
    sc = _StateConfigC(None, 0, None, 0, 0, 0, 1, 1, 0)   # one world, one task graph
    cc = _CompileConfigC(None, 0, None, 0, 1)               # no simulator sources
    h = lib.mb2_executor_create(ctypes.byref(sc), ctypes.byref(cc), 0, None)
    if h:
        lib.mb2_executor_destroy(h)
    return h, (lib.mb2_last_error() or b"").decode()


@pytest.mark.parametrize("knob,value", BAD)
def test_malformed_value_fails_creation(knob_env, knob, value):
    knob_env.setenv("MADRONA_B200_" + knob, value)
    h, msg = _create()
    assert not h
    assert f"MADRONA_B200_{knob} must be " in msg and f'got "{value}"' in msg, msg


@pytest.mark.parametrize("knob,value", GOOD)
def test_valid_value_passes_the_parser(knob_env, knob, value):
    if value is not None:
        knob_env.setenv("MADRONA_B200_" + knob, value)
    h, msg = _create()
    assert not h       # an empty simulator never makes an executor
    assert msg and "MADRONA_B200_" not in msg, msg


def test_valid_cache_dir_passes_the_parser(knob_env, tmp_path):
    knob_env.setenv("MADRONA_B200_KERNEL_CACHE_DIR", str(tmp_path))
    h, msg = _create()
    assert not h
    assert msg and "MADRONA_B200_" not in msg, msg


@pytest.mark.parametrize("knob,value,accepts", [
    ("MAX_HULL_SIZE", "8", "a number from 16 to 255 (vertices and faces per convex hull)"),
    ("MAX_BODIES_PER_WORLD", "", "a number from 128 to 4096 (rigid bodies per world)"),
    ("TMP_BYTES", "256M", f"a number from 1 to {U64_MAX} (bytes of the tmp arena)"),
    ("TABLE_GROWTH", "on", "0 or 1"),
    ("KERNEL_CACHE_DIR", "", "a non-empty path"),
])
def test_error_message(knob_env, knob, value, accepts):
    knob_env.setenv("MADRONA_B200_" + knob, value)
    _, msg = _create()
    assert msg == f'MADRONA_B200_{knob} must be {accepts}, got "{value}"'


@pytest.mark.parametrize("knob,value", [("FAST_MATH", "yes"), ("NO_KERNEL_CACHE", "")])
def test_malformed_value_fails_precompile(knob_env, knob, value):
    knob_env.setenv("MADRONA_B200_" + knob, value)
    with pytest.raises(mb.MadronaB200Error, match=f"MADRONA_B200_{knob} must be 0 or 1"):
        mb.precompile(mb.CompileConfig(userSources=[]))
