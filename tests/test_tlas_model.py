"""CPU checks of the TLAS build rules restated in tests/tlas_model.py: the trees they make
are valid 4-wide BVHs in the ray caster's format (every instance a leaf exactly once,
dequantised child boxes containing their subtree, at most max(1, n - 1) nodes), and the
recorded depth decides whether the traversal stack can hold the tree."""
import numpy as np
import pytest

from tlas_model import MAX_TLAS_DEPTH, build_tlas, decode, quantize_node


def _scattered(n, seed):
    rng = np.random.default_rng(seed)
    c = (rng.random((n, 3)) - 0.5) * np.array([24.0, 24.0, 3.0])
    half = 0.25 + 0.5 * rng.random((n, 3))
    return (c - half).astype(np.float32), (c + half).astype(np.float32)


def _clustered(n):
    # the gallery_sized fixture's clustered layout: radius 6 * 0.93^i, size 1/8 of it
    i = np.arange(n, dtype=np.float64)
    r = 6.0 * 0.93 ** i
    c = np.stack([r * np.cos(2.39996 * i), r * np.sin(2.39996 * i), 2.0 + 0.3 * r], axis=1)
    half = (0.125 * r)[:, None] * np.ones(3)
    return (c - half).astype(np.float32), (c + half).astype(np.float32)


def _check_tree(nodes, depth, lo, hi):
    n = len(lo)
    assert 1 <= len(nodes) <= max(1, n - 1)
    d = decode(nodes)
    seen = np.zeros(n, dtype=np.int64)
    levels = np.zeros(len(nodes), dtype=np.int64)
    levels[0] = 1
    order = []
    stack = [0]
    while stack:
        g = stack.pop()
        order.append(g)
        for c in range(4):
            ch = int(d["children"][g, c])
            if ch == 0xFFFFFFFF:
                assert c >= d["num_children"][g]
                continue
            assert c < d["num_children"][g]
            if ch & 0x80000000:
                seen[ch & 0x7FFFFFFF] += 1
            else:
                assert ch > g                 # canonical numbering: depth first
                levels[ch] = levels[g] + 1
                stack.append(ch)
    assert (seen == 1).all()
    assert depth == levels.max()

    # dequantised child boxes contain every instance box below them
    def instances_below(g):
        out = []
        for c in range(int(d["num_children"][g])):
            ch = int(d["children"][g, c])
            out.append([ch & 0x7FFFFFFF] if ch & 0x80000000 else instances_below(ch))
        return out
    for g in order:
        scale = np.ldexp(np.float32(1), d["exp"][g].astype(np.int32)).astype(np.float64)
        for c, below in enumerate(instances_below(g)):
            below = np.array(_flatten(below))
            qlo = d["min_point"][g].astype(np.float64) + scale * d["qmin"][g, c]
            qhi = d["min_point"][g].astype(np.float64) + scale * d["qmax"][g, c]
            assert (lo[below] >= qlo).all() and (hi[below] <= qhi).all()


def _flatten(x):
    if isinstance(x, list):
        out = []
        for y in x:
            out += _flatten(y)
        return out
    return [x]


@pytest.mark.parametrize("n", [1, 2, 3, 5, 64, 128, 129, 300, 1000])
def test_scattered_trees_are_valid_and_fit_the_stack(n):
    lo, hi = _scattered(n, seed=n)
    nodes, depth = build_tlas(lo, hi)
    _check_tree(nodes, depth, lo, hi)
    assert depth <= MAX_TLAS_DEPTH


def test_many_scattered_instances_fit_the_stack():
    lo, hi = _scattered(9000, seed=1)
    nodes, depth = build_tlas(lo, hi)
    assert len(nodes) <= 8999
    assert depth <= MAX_TLAS_DEPTH


@pytest.mark.parametrize("n", [129, 300])
def test_clustered_trees_are_valid_and_deeper_than_the_stack(n):
    # shrinking clusters share Morton codes: the split falls through the index bits one
    # instance at a time, a tree the ray caster refuses rather than walks with dropped nodes
    lo, hi = _clustered(n)
    nodes, depth = build_tlas(lo, hi)
    _check_tree(nodes, depth, lo, hi)
    assert depth > MAX_TLAS_DEPTH


def test_identical_boxes_still_make_a_tree():
    lo = np.zeros((200, 3), dtype=np.float32)
    hi = np.ones((200, 3), dtype=np.float32)
    nodes, depth = build_tlas(lo, hi)
    _check_tree(nodes, depth, lo, hi)


def test_quantize_node_contains_children():
    rng = np.random.default_rng(7)
    for _ in range(200):
        k = int(rng.integers(1, 5))
        base = (rng.random(3) - 0.5) * 10.0 ** rng.integers(-3, 4)
        cmin = (base + rng.random((k, 3)) * 10.0 ** rng.integers(-4, 3)).astype(np.float32)
        cmax = (cmin + rng.random((k, 3)) * 10.0 ** rng.integers(-4, 3)).astype(np.float32)
        raw = np.frombuffer(bytes(quantize_node(cmin, cmax)), dtype=np.uint8).reshape(1, 60)
        d = decode(raw)
        assert d["num_children"][0] == k
        scale = np.ldexp(np.float32(1), d["exp"][0].astype(np.int32)).astype(np.float64)
        for c in range(k):
            qlo = d["min_point"][0].astype(np.float64) + scale * d["qmin"][0, c]
            qhi = d["min_point"][0].astype(np.float64) + scale * d["qmax"][0, c]
            assert (cmin[c] >= qlo).all() and (cmax[c] <= qhi).all()
