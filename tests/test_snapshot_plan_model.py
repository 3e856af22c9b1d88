"""Segment plan and chunk walk of the snapshot copy kernel (madrona_b200/csrc/kernels_snapshot.cu),
modelled on the CPU: segments laid out in the snapshot buffer as the host planner lays them
out, chunks found by the kernel's binary search, each chunk copied with the kernel's 16-byte /
4-byte / byte split and its thread-to-unit mapping.  For row counts of 0, 1 and around chunk
edges, rows of 4, 12, 24, 28 and 96 bytes and live bases that are not 16-byte aligned, every
byte of every segment's live rows must be copied exactly once, in both directions, and no
byte outside them written."""
import os
import re

import numpy as np
import pytest

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                   "madrona_b200", "csrc", "kernels_snapshot.cu")


def _constant(name):
    text = open(SRC).read()
    m = re.search(r"constexpr int " + name + r" = (\d+);", text)
    assert m, name
    return int(m.group(1))


THREADS = _constant("kSnapThreads")
UNITS = _constant("kSnapUnitsPerThread")
CHUNK = THREADS * UNITS * 16


def plan(segments):
    """Host planner: snapshot offsets (256-byte aligned regions of >= 256 bytes, else 16) and
    each segment's first chunk.  segments: dicts with rows (capacity) and row_bytes."""
    offset = chunks = 0
    out = []
    for s in segments:
        nbytes = s["rows"] * s["row_bytes"]
        if nbytes <= 0:
            continue
        align = 256 if nbytes >= 256 else 16
        offset = (offset + align - 1) // align * align
        out.append(dict(s, snap=offset, first_chunk=chunks))
        offset += nbytes
        chunks += (nbytes + CHUNK - 1) // CHUNK
    return out, offset, chunks


def find_segment(segs, c):
    lo, hi = 0, len(segs) - 1
    while lo < hi:
        mid = (lo + hi + 1) >> 1
        if segs[mid]["first_chunk"] <= c:
            lo = mid
        else:
            hi = mid - 1
    return lo


def copy_chunk(src_mem, src, dst_mem, dst, length, writes):
    """snapCopyChunk: which thread copies which bytes does not matter for the result, but
    the 16-byte units must all be reached by the (thread, k) mapping"""
    def move(lo, hi):
        dst_mem[dst + lo:dst + hi] = src_mem[src + lo:src + hi]
        writes[dst + lo:dst + hi] += 1

    done = 0
    if (src | dst) & 15 == 0:
        n = length >> 4
        reached = np.zeros(n, dtype=np.int32)
        for k in range(UNITS):
            units = np.arange(THREADS) + k * THREADS
            np.add.at(reached, units[units < n], 1)
        assert (reached == 1).all()
        move(0, n << 4)
        done = n << 4
    if ((src + done) | (dst + done)) & 3 == 0:
        n = (length - done) >> 2
        move(done, done + (n << 2))
        done += n << 2
    move(done, length)


def run_kernel(segs, num_chunks, live_mem, snap_mem, live_counts, snap_counts, restore, writes, grid=7):
    for b in range(grid):
        for c in range(b, num_chunks, grid):
            g = segs[find_segment(segs, c)]
            count = (snap_counts if restore else live_counts)[g["name"]]
            rows = g["rows"] if count is None else max(0, min(count, g["rows"]))
            nbytes = rows * g["row_bytes"]
            off = (c - g["first_chunk"]) * CHUNK
            if off >= nbytes:
                continue
            length = min(nbytes - off, CHUNK)
            if restore:
                copy_chunk(snap_mem, g["snap"] + off, live_mem, g["live"] + off, length, writes)
            else:
                copy_chunk(live_mem, g["live"] + off, snap_mem, g["snap"] + off, length, writes)


def layout(specs, misalign):
    """Live addresses: each segment at a 256-byte boundary plus its misalignment, 64 guard
    bytes after its capacity."""
    segs, addr = [], 0
    for i, (rows, row_bytes, count) in enumerate(specs):
        addr = (addr + 255) // 256 * 256 + misalign[i % len(misalign)]
        segs.append({"name": i, "rows": rows, "row_bytes": row_bytes, "live": addr, "count": count})
        addr += rows * row_bytes + 64
    return segs, addr + 256


def edge_rows(row_bytes):
    per_chunk = CHUNK // row_bytes
    return sorted({0, 1, 2, per_chunk - 1, per_chunk, per_chunk + 1, 2 * per_chunk + 3})


CASES = []
for rb in (4, 12, 24, 28, 96):
    for mis in ((0,), (4,), (0, 4, 8, 12), (1, 3)):
        CASES.append((rb, mis))


@pytest.mark.parametrize("row_bytes,misalign", CASES)
def test_every_live_byte_is_copied_once_and_nothing_else(row_bytes, misalign):
    rng = np.random.default_rng(row_bytes * 31 + sum(misalign))
    specs = []
    for n in edge_rows(row_bytes):
        cap = n + int(rng.integers(0, 40))
        specs.append((max(cap, 1), row_bytes, n))             # a device-known count
    specs.append((37, row_bytes, None))                       # a fixed count
    specs.append((5, row_bytes, 9))                           # a count past the capacity: clamped
    specs.append((5, row_bytes, -3))                          # a negative count: nothing
    specs.append((1, 12, None))                               # scalars
    specs.append((1, 8, None))
    segs, live_size = layout(specs, misalign)
    planned, snap_size, num_chunks = plan(segs)
    counts = {s["name"]: s["count"] for s in segs}
    live = rng.integers(0, 256, size=live_size, dtype=np.uint8)
    snap = np.zeros(snap_size + 256, dtype=np.uint8)

    def live_span(g):
        c = counts[g["name"]]
        rows = g["rows"] if c is None else max(0, min(c, g["rows"]))
        return rows * g["row_bytes"]

    # save: every live byte lands once in the segment's region of the snapshot
    writes = np.zeros_like(snap, dtype=np.int32)
    run_kernel(planned, num_chunks, live, snap, counts, None, False, writes)
    want = np.zeros_like(writes)
    for g in planned:
        n = live_span(g)
        want[g["snap"]:g["snap"] + n] = 1
        assert np.array_equal(snap[g["snap"]:g["snap"] + n], live[g["live"]:g["live"] + n])
    assert np.array_equal(writes, want)
    # regions never overlap and keep their alignment
    for a, b in zip(planned, planned[1:]):
        assert a["snap"] + a["rows"] * a["row_bytes"] <= b["snap"]
    assert all(g["snap"] % 16 == 0 for g in planned)

    # restore over different live bytes, reading the counts the snapshot holds
    saved = live.copy()
    live2 = rng.integers(0, 256, size=live_size, dtype=np.uint8)
    before = live2.copy()
    live_counts_now = {k: None if v is None else v + 5 for k, v in counts.items()}   # what it overwrites
    writes = np.zeros(live_size, dtype=np.int32)
    run_kernel(planned, num_chunks, live2, snap, live_counts_now, counts, True, writes)
    want = np.zeros_like(writes)
    for g in planned:
        n = live_span(g)
        want[g["live"]:g["live"] + n] = 1
    assert np.array_equal(writes, want)
    assert np.array_equal(live2[want == 1], saved[want == 1])
    assert np.array_equal(live2[want == 0], before[want == 0])


def test_chunk_is_what_one_block_moves_in_one_pass():
    assert CHUNK == THREADS * UNITS * 16
    assert CHUNK % 256 == 0
