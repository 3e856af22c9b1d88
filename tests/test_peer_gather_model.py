"""CPU model of the peer-store gather (madrona_b200/csrc/peer_gather.cu): the push kernel's
store plan at every rank of 1 to kMaxPeers ranks, and the push / wait / release flag protocol
of ranks that share one stream (how tests/test_peer_gather.py runs N ranks on one GPU).

The store plan restates gatherPushKernel and mb2_peer_gather_push_async: the grid, the
grid-stride loop over a slot's whole 16-byte vectors, the peer rotation of each vector's
stores, the store width and the 1 to 3 word tail.  The flag protocol restates the spin
conditions of the push, wait and release kernels.  No GPU needed."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gather_constant(name):
    src = open(os.path.join(ROOT, "madrona_b200", "csrc", "peer_gather.cu")).read()
    m = re.search(r"constexpr int " + name + r" = (\d+);", src)
    assert m, name
    return int(m.group(1))


MAX_SLOTS = _gather_constant("kMaxGatherSlots")
MAX_PEERS = _gather_constant("kMaxPeers")
THREADS = 256            # gatherPushKernel's block (__launch_bounds__(256), push_async)
MAX_BLOCKS = 32          # push_async's grid cap

# slice sizes (bytes of one rank's column): every residue mod 16, tail-only slices, one and
# several grid-stride passes of the 32-block grid
SIZES = [4, 8, 12, 16, 20, 28, 40, 1028, 4112, 8184, 131072, 131084, 261888]


def _layouts():
    """Slot lists of 1 to MAX_SLOTS slots that take SIZES in turn, so every size sits in
    several slot positions and next to both small and large slots."""
    out, at = [], 0
    for n in range(1, MAX_SLOTS + 1):
        out.append([SIZES[(at + j) % len(SIZES)] for j in range(n)])
        at += n
    return out


LAYOUTS = _layouts()


def buffer_layout(slot_bytes, world_size):
    """mb2_peer_gather_create: each slot's offset inside a parity ([world_size][bytes],
    rounded up to 256 bytes) and the bytes of one parity."""
    offsets, off = [], 0
    for b in slot_bytes:
        offsets.append(off)
        off += (b * world_size + 255) & ~255
    return offsets, off


def push_grid(slot_bytes):
    """mb2_peer_gather_push_async: blocks of the push kernel."""
    return max(1, min((max(slot_bytes) // 16 + 255) // 256, MAX_BLOCKS))


def store_width(dst_off):
    """The widest store a slice starting at dst_off allows (the same on every peer)."""
    return 16 if dst_off % 16 == 0 else 8 if dst_off % 8 == 0 else 4


def store_width_16_only(dst_off):
    """The plan before slices of any multiple of 4 were supported: always 16-byte stores."""
    return 16


def push_plan(slot_bytes, world_size, rank, step, width_of=store_width):
    """Every store one push kernel makes, per slot: (peer [n], destination byte offset in that
    peer's buffer [n], source byte offset in the slot's column [n], width).  The vector part
    is one row per vector and one column per iteration k of the peer loop."""
    P = world_size
    offsets, parity_bytes = buffer_layout(slot_bytes, P)
    stride = push_grid(slot_bytes) * THREADS
    plan = []
    for s, b in enumerate(slot_bytes):
        vecs = b >> 4
        dst_off = (step & 1) * parity_bytes + offsets[s] + rank * b
        w = width_of(dst_off)
        # the grid-stride loop: global thread t takes vectors t, t + stride, ...
        passes = -(-vecs // stride)
        i = (np.arange(stride)[None, :] + stride * np.arange(passes)[:, None]).ravel()
        i = i[i < vecs]
        k = np.arange(P)
        peer = (k[None, :] + rank + 1 + (i[:, None] >> 5)) % P                 # [vectors, k]
        sub = np.arange(16 // w) * w
        src = (16 * i[:, None] + sub[None, :])                                  # [vectors, stores]
        vec = (np.broadcast_to(peer[:, :, None], peer.shape + (sub.size,)),
               np.broadcast_to(src[:, None, :], peer.shape + (sub.size,)))
        # the tail: block 0's first (bytes & 15) / 4 threads, one word each to every peer
        tail_src = 16 * vecs + 4 * np.arange((b & 15) >> 2)
        tail = (np.repeat(np.arange(P), tail_src.size), np.tile(tail_src, P))
        plan.append({"slot": s, "dst_off": dst_off, "width": w, "vec_peer": vec[0], "vec_src": vec[1],
                     "vectors": i, "tail_peer": tail[0], "tail_src": tail[1]})
    return plan


def misaligned_stores(plan):
    return sum(int(((p["dst_off"] + p["vec_src"]) % p["width"] != 0).sum()) +
               int(((p["dst_off"] + p["tail_src"]) % 4 != 0).sum()) for p in plan)


def check_store_plan(slot_bytes, P):
    """Push steps 0 and 1 (both parities) of every rank and check every peer's buffer: each
    byte of each rank's slice lands exactly once, holds the byte it should, and nothing
    outside the slices is written; every store is aligned to its width."""
    offsets, parity_bytes = buffer_layout(slot_bytes, P)
    words = 2 * parity_bytes // 4
    # word value: which (step, rank, slot, source word) it came from
    tag_stride = max(slot_bytes) // 4

    def tag(step, rank, slot, src_word):
        return ((step * P + rank) * MAX_SLOTS + slot) * tag_stride + src_word

    want = np.full(words, -1, dtype=np.int64)
    for step in (0, 1):
        for r in range(P):
            for s, b in enumerate(slot_bytes):
                first = (step * parity_bytes + offsets[s] + r * b) // 4
                want[first:first + b // 4] = tag(step, r, s, np.arange(b // 4))

    stores = []           # word index (peer * words + word) of every word stored
    got = np.full(P * words, -1, dtype=np.int64)
    for step in (0, 1):
        for r in range(P):
            for p in push_plan(slot_bytes, P, r, step):
                b = slot_bytes[p["slot"]]
                assert misaligned_stores([p]) == 0, (P, r, b, p["width"])
                # the grid-stride loop visits every vector once
                assert np.array_equal(np.sort(p["vectors"]), np.arange(b >> 4)), (P, r, b)
                w = p["width"]
                for peer, src, width in ((p["vec_peer"], p["vec_src"], w), (p["tail_peer"], p["tail_src"], 4)):
                    peer, src = peer.ravel(), src.ravel()
                    # every store as its words
                    sw = (src[:, None] // 4 + np.arange(width // 4)[None, :]).ravel()
                    pw = np.repeat(peer, width // 4)
                    at = pw * words + (p["dst_off"] // 4) + sw
                    stores.append(at)
                    got[at] = tag(step, r, p["slot"], sw)
    count = np.bincount(np.concatenate(stores), minlength=P * words).reshape(P, words)
    got = got.reshape(P, words)
    inside = want >= 0
    assert (count[:, inside] == 1).all(), f"a slice byte lands twice or never: P={P} {slot_bytes}"
    assert (count[:, ~inside] == 0).all(), f"a store outside the slices: P={P} {slot_bytes}"
    assert (got == want[None, :]).all(), f"a slice byte holds the wrong source byte: P={P} {slot_bytes}"


def test_constants_read_from_the_kernel():
    assert MAX_SLOTS >= 1 and MAX_PEERS >= 1
    assert len(LAYOUTS) == MAX_SLOTS and max(len(lay) for lay in LAYOUTS) == MAX_SLOTS
    assert sorted({b for lay in LAYOUTS for b in lay}) == sorted(SIZES)


@pytest.mark.parametrize("P", range(1, MAX_PEERS + 1))
def test_push_stores_every_slice_byte_once_at_its_offset(P):
    for slot_bytes in LAYOUTS:
        check_store_plan(slot_bytes, P)


def test_store_width_follows_the_slice_alignment():
    # rank r of 1028-byte slices starts at r * 1028 = 4 r (mod 16): 16, 4, 8, 4, 16, ...
    widths = [store_width(r * 1028) for r in range(MAX_PEERS)]
    assert widths[:5] == [16, 4, 8, 4, 16]
    # 16-byte multiples (the benchmark's columns) keep 16-byte stores at every rank
    for b in (8192 * 4, 4096 * 8, 4112, 131072):
        assert {store_width(r * b) for r in range(MAX_PEERS)} == {16}


def test_16_byte_only_plan_misaligns_rank_1_of_1028_byte_slices():
    """The finding behind the store widths: with 16-byte stores only, rank 1 of 2 ranks of
    257 cartpole worlds (a 1028-byte reward column) stores at byte 1028 of every peer's
    buffer, 4 bytes off a 16-byte boundary."""
    assert misaligned_stores(push_plan([1028], 2, 0, 0, store_width_16_only)) == 0
    bad = misaligned_stores(push_plan([1028], 2, 1, 0, store_width_16_only))
    assert bad == 2 * (1028 // 16)        # every vector store, to both peers
    assert misaligned_stores(push_plan([1028], 2, 1, 0)) == 0
    # slices of 16-byte multiples are aligned under both plans
    for r in range(4):
        assert misaligned_stores(push_plan([32768, 32768], 4, r, 0, store_width_16_only)) == 0


# ---- flag protocol ---------------------------------------------------------------------------


class Spin(AssertionError):
    """A spin kernel whose condition does not hold when it starts: on one stream nothing else
    can run behind it, so it would spin forever."""


class GatherModel:
    """N ranks' gathers on one stream: each kernel runs to completion in issue order."""

    def __init__(self, n):
        self.n = n
        self.push_step = [0] * n
        self.wait_step = [0] * n
        self.release_step = [0] * n
        # flags block of rank r: arrived[q], released[q] (written by rank q)
        self.arrived = [[0] * n for _ in range(n)]
        self.released = [[0] * n for _ in range(n)]
        # buffer of rank r: [parity][q] = (step, q) of the data that sits there
        self.buffer = [[[None] * n for _ in range(2)] for _ in range(n)]
        self.column = [None] * n            # what rank r's step graph exported last

    def run(self, r, k):
        self.column[r] = (k, r)

    def push(self, r):
        step = self.push_step[r]
        if step >= 2 and any(self.released[r][q] < step - 1 for q in range(self.n)):
            raise Spin(f"push({step}) of rank {r}: released {self.released[r]}")
        for p in range(self.n):
            self.buffer[p][step & 1][r] = self.column[r]
            self.arrived[p][r] = step + 1
        self.push_step[r] = step + 1

    def wait(self, r):
        step = self.wait_step[r]
        if any(self.arrived[r][q] < step + 1 for q in range(self.n)):
            raise Spin(f"wait({step}) of rank {r}: arrived {self.arrived[r]}")
        self.wait_step[r] = step + 1

    def read(self, r, k):
        """What rank r reads from its gathered buffer of step k (parity k & 1)."""
        assert self.wait_step[r] == k + 1 and self.release_step[r] == k
        return list(self.buffer[r][k & 1])

    def release(self, r):
        step = self.release_step[r]
        for p in range(self.n):
            self.released[p][r] = step + 1
        self.release_step[r] = step + 1


def run_issue_order(n, steps, skip_release=None):
    """bench.py's order, as tests/test_peer_gather.py issues it on one stream: for each rank
    run(k) and push(k), then for each rank wait(k - 1), read, release(k - 1); a final
    wait / read / release of the last step.  Returns every read."""
    m = GatherModel(n)
    reads = []

    def consume(k):
        for r in range(n):
            m.wait(r)
            reads.append((r, k, m.read(r, k)))
            if (r, k) != skip_release:
                m.release(r)

    for k in range(steps):
        for r in range(n):
            m.run(r, k)
            m.push(r)
        if k >= 1:
            consume(k - 1)
    consume(steps - 1)
    return reads


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8, 16])
def test_issue_order_never_spins_and_reads_its_own_step(n):
    assert n <= MAX_PEERS
    steps = 12
    reads = run_issue_order(n, steps)
    assert len(reads) == n * steps
    for r, k, got in reads:
        # step k of every rank, from parity k & 1: never step k + 2 (the next user of the parity)
        assert got == [(k, q) for q in range(n)], (r, k, got)


@pytest.mark.parametrize("n", [2, 3, 16])
def test_model_refuses_orders_that_would_spin_forever(n):
    # the loop-back order (push(k), then wait(k) at once) only works for one rank: rank 0
    # would wait for the push of rank 1, which sits behind it on the stream
    m = GatherModel(n)
    m.run(0, 0)
    m.push(0)
    with pytest.raises(Spin):
        m.wait(0)
    # a rank that never releases step 2 holds back every push of step 4
    with pytest.raises(Spin):
        run_issue_order(n, 12, skip_release=(n - 1, 2))


def test_loopback_order_of_one_rank():
    m = GatherModel(1)
    for k in range(6):
        m.run(0, k)
        m.push(0)
        m.wait(0)
        assert m.read(0, k) == [(k, 0)]
        m.release(0)
