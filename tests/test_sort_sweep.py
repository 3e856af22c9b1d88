"""Archetype sort and compaction (kernels_sort.cu) against a stable-sort model, at the
edges where the kernels change behaviour:

- row counts around the 2048-row tile / rearrange chunk, more tiles than the 8-tile
  look-back window, one digit holding every row, keys of 0xFFFFFFFF (kept by a custom sort);
- a key column wider than 4 bytes (pass 0 reads it row by row instead of by TMA);
- 1/2/3/5/6/8/12/20/24/32/48-byte columns (uchar, ushort, uint, uint2, uint4 units, power
  of two and not), exported ones (copied back) and non-exported ones (flipped);
- world counts where the world sort's pass count changes (255/256, 65535/65536), empty
  worlds, steps that delete whole worlds or the whole table, a custom sort over destroyed
  rows followed by a compaction, and tables that grow between steps.

The fixture (sims/sortsweep) makes every byte of a row a pure function of (world, uid,
component, byte) and every key a pure function of (seed, uid, step).  The model here holds
the table as (world, uid, key, alive) rows, applies the fixture's churn and each sort
through oracle/restate.sort_archetype; it is itself checked against a naive per-world
list simulation.  Every comparison is exact.
"""
import numpy as np
import pytest

from oracle import restate

M32 = 0xFFFFFFFF
ALL_ONES = np.uint64(M32)
SHAPE_SORT, SHAPE_CHURN, SHAPE_REKEY_CHURN_SORT = 0, 1, 2
KEY_UNIFORM, KEY_CONSTANT, KEY_ALL_ONES, KEY_BYTE3 = 0, 1, 2, 3
WIDTHS = [1, 2, 3, 5, 8, 12, 20, 24, 32, 48, 6]      # payload component c has WIDTHS[c] bytes
# export slot -> payload component index (sims/sortsweep/sim.hpp ExportID)
EXPORTED_PAYLOADS = {4: 1, 5: 2, 6: 5, 7: 7, 8: 9}
SLOT_ENTITY, SLOT_UID, SLOT_KEY4, SLOT_CHECK, SLOT_SUMMARY = 0, 1, 2, 3, 9
TILE = 2048


# ---- the fixture's pure functions (sims/sortsweep/sim.hpp), on uint64 arrays holding uint32 values ----

def _u(x):
    return np.asarray(x, dtype=np.uint64) & np.uint64(M32)


def mix32(h):
    h = _u(h)
    h ^= h >> np.uint64(16)
    h = (h * np.uint64(0x85EBCA6B)) & np.uint64(M32)
    h ^= h >> np.uint64(13)
    h = (h * np.uint64(0xC2B2AE35)) & np.uint64(M32)
    h ^= h >> np.uint64(16)
    return h


def hash_of(seed, uid, t):
    inner = mix32(_u(uid) * np.uint64(0x9E3779B1) + _u(t) * np.uint64(0x7F4A7C15) + np.uint64(1))
    return mix32(_u(seed) ^ inner)


def key_of(seed, uid, t, mode):
    r = hash_of(_u(seed) ^ np.uint64(0x5BD1E995), uid, t)
    if mode == KEY_CONSTANT:
        return np.full_like(r, 0x2A2A2A2A)
    if mode == KEY_ALL_ONES:
        return np.full_like(r, M32)
    if mode == KEY_BYTE3:
        return r & np.uint64(0xFF000000)
    return np.where((r & np.uint64(0xF)) == 0, ALL_ONES, r)


def payload_bytes(world, uid, c):
    """(rows, WIDTHS[c]) uint8: byte i of payload c of each row."""
    row = mix32(_u(uid) * np.uint64(0x9E3779B1) + _u(world) * np.uint64(0x85EBCA77) + np.uint64(1))
    h = mix32(row + np.uint64(c) * np.uint64(0x27D4EB2F))
    i = np.arange(WIDTHS[c], dtype=np.uint64)
    return (((h[:, None] >> (np.uint64(8) * (i & np.uint64(3)))) + np.uint64(0x3B) * (i >> np.uint64(2)))
            & np.uint64(0xFF)).astype(np.uint8)


def summary_term(uid, i):
    return mix32(_u(uid) + _u(i) * np.uint64(0x9E3779B9))


# ---- the model ----

class Model:
    """The Item table as global rows (world, uid, key, alive) in table order; `ent` rides along
    (the entity the GPU reported for the row, -1 until seen)."""

    def __init__(self, cfg):
        self.W = len(cfg["init_counts"])
        self.seeds = np.arange(self.W, dtype=np.uint64) + np.uint64(cfg.get("seed", 0))
        self.creates = np.asarray(cfg["creates"], dtype=np.int64)
        self.kill = np.asarray(cfg["kill_steps"], dtype=np.int64)
        self.shape, self.mode = cfg["shape"], cfg["key_mode"]
        self.threshold = np.uint64(cfg["destroy_threshold"])
        counts = np.asarray(cfg["init_counts"], dtype=np.int64)
        self.next_uid = counts.copy()
        # construction appends each world's items in creation order; the initial world sort keeps it
        self.world = np.repeat(np.arange(self.W, dtype=np.int64), counts)
        self.uid = np.arange(len(self.world), dtype=np.int64) - np.repeat(np.cumsum(counts) - counts, counts)
        self.key = key_of(self.seeds[self.world], self.uid, 0, self.mode)
        self.alive = np.ones(len(self.world), dtype=bool)
        self.ent = np.full(len(self.world), -1, dtype=np.int64)
        self.t = 0
        self.offsets = self.counts = None

    @property
    def n(self):
        return len(self.world)

    def _apply(self, perm):
        for name in ("world", "uid", "key", "alive", "ent"):
            setattr(self, name, getattr(self, name)[perm])

    def step(self):
        self.t = t = self.t + 1
        if self.shape != SHAPE_CHURN:
            self.key = key_of(self.seeds[self.world], self.uid, t, self.mode)
        if self.shape != SHAPE_SORT:
            die = (self.kill[self.world] == t) | (hash_of(self.seeds[self.world], self.uid, t) < self.threshold)
            self.alive &= ~die
            made = np.where(self.kill == t, 0, self.creates)
            world = np.repeat(np.arange(self.W, dtype=np.int64), made)
            uid = self.next_uid[world] + (np.arange(len(world)) - np.repeat(np.cumsum(made) - made, made))
            self.next_uid += made
            key_t = 0 if self.shape == SHAPE_CHURN else t
            self.world = np.concatenate([self.world, world])
            self.uid = np.concatenate([self.uid, uid])
            self.key = np.concatenate([self.key, key_of(self.seeds[world], uid, key_t, self.mode)])
            self.alive = np.concatenate([self.alive, np.ones(len(world), dtype=bool)])
            self.ent = np.concatenate([self.ent, np.full(len(world), -1, dtype=np.int64)])
        if self.shape != SHAPE_CHURN:
            perm, _, _, _ = restate.sort_archetype(self.key.astype(np.uint32), self.W, world_sort=False)
            self._apply(perm)
        if self.shape != SHAPE_SORT:
            self.world_keys = wkey = np.where(self.alive, self.world, M32).astype(np.uint32)
            perm, _, self.offsets, self.counts = restate.sort_archetype(wkey, self.W, world_sort=True)
            self._apply(perm)

    def summary(self):
        """(W, 2) uint32: per world (row count, sum of summary_term(uid, position in world))."""
        pos = np.arange(self.n, dtype=np.int64) - self.offsets[self.world]
        term = summary_term(self.uid, pos)
        h = np.zeros(self.W, dtype=np.uint64)
        np.add.at(h, self.world, term)
        return np.stack([self.counts.astype(np.uint64), h & np.uint64(M32)], axis=1).astype(np.uint32)


def naive_run(cfg, steps):
    """Per-world Python lists, sorted with Python's stable sort: [(world, uid, key)] per step, plus
    (offsets, counts) where the step compacts."""
    W = len(cfg["init_counts"])
    seed0, shape, mode = cfg.get("seed", 0), cfg["shape"], cfg["key_mode"]
    thr = cfg["destroy_threshold"]

    def key(w, u, t):
        return int(key_of(seed0 + w, u, t, mode))

    worlds = [[[u, key(w, u, 0), True] for u in range(cfg["init_counts"][w])] for w in range(W)]
    next_uid = list(cfg["init_counts"])
    table = [(w, r[0], r[1]) for w in range(W) for r in worlds[w]]   # shape SORT keeps one global list
    out = []
    for t in range(1, steps + 1):
        if shape == SHAPE_SORT:
            table = sorted([(w, u, key(w, u, t)) for (w, u, _) in table], key=lambda r: r[2])
            out.append((table, None))
            continue
        rows = []
        for w in range(W):
            lst = worlds[w]
            for r in lst:
                if shape == SHAPE_REKEY_CHURN_SORT:
                    r[1] = key(w, r[0], t)
                if cfg["kill_steps"][w] == t or int(hash_of(seed0 + w, r[0], t)) < thr:
                    r[2] = False
            if cfg["kill_steps"][w] != t:
                for _ in range(cfg["creates"][w]):
                    lst.append([next_uid[w], key(w, next_uid[w], 0 if shape == SHAPE_CHURN else t), True])
                    next_uid[w] += 1
            if shape == SHAPE_REKEY_CHURN_SORT:
                lst.sort(key=lambda r: r[1])
            worlds[w] = [r for r in lst if r[2]]
            rows += [(w, r[0], r[1]) for r in worlds[w]]
        counts = [len(worlds[w]) for w in range(W)]
        starts = np.cumsum([0] + counts[:-1])
        offsets = [int(starts[w]) if counts[w] else len(rows) for w in range(W)]
        out.append((rows, (offsets, counts)))
    return out


def _random_cfg(rng):
    W = int(rng.integers(1, 7))
    cfg = {"shape": int(rng.integers(0, 3)), "key_mode": int(rng.integers(0, 4)), "seed": int(rng.integers(0, 1000)),
           "destroy_threshold": int(rng.choice([0, 1 << 30, 1 << 31, M32])),
           "init_counts": [int(x) for x in rng.integers(0, 9, W)],
           "creates": [int(x) for x in rng.integers(0, 4, W)],
           "kill_steps": [int(x) for x in rng.integers(0, 6, W)]}
    if cfg["shape"] == SHAPE_SORT:
        cfg["creates"], cfg["kill_steps"], cfg["destroy_threshold"] = [0] * W, [0] * W, 0
    return cfg


# ---- CPU tests: the model itself ----

@pytest.mark.parametrize("script", range(40))
def test_model_matches_naive_per_world_lists(script):
    cfg = _random_cfg(np.random.default_rng(1000 + script))
    steps = 6
    model = Model(cfg)
    for t, (rows, summary) in enumerate(naive_run(cfg, steps), start=1):
        model.step()
        got = list(zip(model.world.tolist(), model.uid.tolist(), model.key.tolist()))
        assert got == rows, (cfg, t)
        if summary is not None:
            assert model.offsets.tolist() == summary[0] and model.counts.tolist() == summary[1], (cfg, t)


def test_model_keeps_all_ones_custom_keys_and_drops_only_destroyed_rows():
    cfg = {"shape": SHAPE_SORT, "key_mode": KEY_ALL_ONES, "destroy_threshold": 0, "init_counts": [3, 0, 2],
           "creates": [0, 0, 0], "kill_steps": [0, 0, 0]}
    model = Model(cfg)
    model.step()
    assert model.n == 5 and model.uid.tolist() == [0, 1, 2, 0, 1]


def _rows_kept_by_world_sort(world_keys, passes):
    """Rows an LSD world sort on the low 8*passes key bits keeps, in order (destroyed rows are
    counted on the full key and cut from the end)."""
    mask = np.uint32((1 << (8 * passes)) - 1) if passes < 4 else np.uint32(M32)
    keep = int((world_keys != np.uint32(M32)).sum())
    return np.argsort(world_keys & mask, kind="stable")[:keep]


@pytest.mark.parametrize("W", [256, 257, 65536, 65537])
def test_churn_cases_tell_one_radix_pass_too_few_apart(W):
    # At W = 256 / 65536 the world sort needs one more radix pass than at W - 1.  With one pass
    # too few, world W - 1's low digits equal those of a destroyed row's all-ones key, so the
    # GPU churn cases below must give that world rows while other worlds destroy some.
    cfg = _churn_cfg(W)
    model = Model(cfg)
    passes = restate.world_sort_passes(W)
    assert passes == (2 if W < 65536 else 3)
    differs = False
    for _ in range(4):
        model.step()
        assert model.counts[W - 1] > 0
        right = _rows_kept_by_world_sort(model.world_keys, passes)
        assert np.array_equal(model.world, model.world_keys[right].astype(np.int64))
        differs |= not np.array_equal(right, _rows_kept_by_world_sort(model.world_keys, passes - 1))
    assert differs


def test_generators_match_known_values():
    # values printed by the same functions compiled as C++ (sims/sortsweep/sim.hpp)
    assert int(mix32(0)) == 0 and int(mix32(1)) == 0x514E28B7 and int(mix32(0xDEADBEEF)) == 0x0DE5C6A9
    assert int(hash_of(7, 3, 2)) == 0x109E62EE
    assert [int(key_of(7, 3, 2, m)) for m in range(4)] == [0x98DEFE8F, 0x2A2A2A2A, 0xFFFFFFFF, 0x98000000]
    assert int(key_of(1, 9, 1, KEY_UNIFORM)) == M32          # a uniform key forced to all-ones
    p48 = payload_bytes(np.array([5]), np.array([11]), 9)[0]
    assert p48[:8].tolist() == [0x65, 0x3A, 0x7D, 0xA7, 0xA0, 0x75, 0xB8, 0xE2]
    assert p48[40:].tolist() == [0xB3, 0x88, 0xCB, 0xF5, 0xEE, 0xC3, 0x06, 0x30]
    assert int(summary_term(11, 4)) == 0xED77732D


# ---- GPU tests ----

def _uneven(total, W, rng, empty_every=0):
    """W non-negative counts summing to `total`, uneven, every `empty_every`-th world empty."""
    weights = rng.random(W) ** 3 + 1e-3
    if empty_every:
        weights[::empty_every] = 0
    counts = np.floor(weights / weights.sum() * total).astype(np.int64)
    counts[int(np.argmax(weights))] += total - counts.sum()
    return [int(c) for c in counts]


def _fetch(ex, slot, dtype, n, width):
    return ex.tensor(slot, dtype, (n, width)).cpu().numpy()


def _check_step(ex, model, step):
    n = model.n
    for slot in (SLOT_ENTITY, SLOT_UID, SLOT_KEY4, SLOT_CHECK, *EXPORTED_PAYLOADS):
        assert ex.exportedNumRows(slot) == n, (step, slot, ex.exportedNumRows(slot), n)
    if model.shape != SHAPE_SORT:
        summary = _fetch(ex, SLOT_SUMMARY, "uint32", model.W, 2)
        want = model.summary()
        bad = np.flatnonzero((summary != want).any(axis=1))
        assert bad.size == 0, f"step {step}: world {bad[0]} summary {summary[bad[0]]} != {want[bad[0]]}"
    if n == 0:
        return

    def first_bad(ok, what):
        if not ok.all():
            r = int(np.flatnonzero(~ok)[0])
            raise AssertionError(f"step {step}: {what} differs first at row {r} of {n} "
                                 f"(world {model.world[r]}, uid {model.uid[r]})")

    check = _fetch(ex, SLOT_CHECK, "uint32", n, 1)[:, 0]
    first_bad(check == 0, f"device check (mismatch bits {check[check != 0][:1]})")
    uid = _fetch(ex, SLOT_UID, "uint32", n, 1)[:, 0]
    first_bad(uid == model.uid, "Uid")
    key = _fetch(ex, SLOT_KEY4, "uint32", n, 1)[:, 0]
    first_bad(key == model.key, "Key4")

    ent = _fetch(ex, SLOT_ENTITY, "int32", n, 2)
    gen, eid = ent[:, 0].astype(np.uint32).astype(np.int64), ent[:, 1].astype(np.int64)
    first_bad((eid >= 0) & (gen != M32), "Entity (a destroyed or missing entity)")
    assert np.unique(eid).size == n, f"step {step}: an entity id appears on two rows"
    packed = (gen << 32) | eid
    known = model.ent >= 0
    first_bad(~known | (packed == model.ent), "Entity (a row's entity changed)")
    model.ent = packed

    # exported payloads, byte for byte (a sample of rows on the largest tables; the device
    # check above covers every byte of every row)
    rows = np.arange(n)
    if n > 300_000:
        rows = np.unique(np.concatenate([rows[:8192], rows[-8192:], rows[::61]]))
    for slot, c in EXPORTED_PAYLOADS.items():
        got = _fetch(ex, slot, "uint8", n, WIDTHS[c])[rows]
        want = payload_bytes(model.world[rows], model.uid[rows], c)
        ok = np.ones(n, dtype=bool)
        ok[rows] = (got == want).all(axis=1)
        first_bad(ok, f"{WIDTHS[c]}-byte exported payload")


def _run_case(cfg, steps, expect_rows=None):
    from sims import make_executor
    model = Model(cfg)
    if expect_rows is not None:
        assert model.n == expect_rows
    ex = make_executor("sortsweep", model.W, **cfg)
    try:
        graph = ex.buildLaunchGraphAllTaskGraphs()
        ptrs = [ex.getExported(s) for s in range(10)]
        for step in range(1, steps + 1):
            ex.run(graph)
            model.step()
            _check_step(ex, model, step)
            assert [ex.getExported(s) for s in range(10)] == ptrs, f"step {step}: an exported column moved"
    finally:
        ex.close()
    return model


def _sort_cfg(counts, mode, key8, seed=17):
    W = len(counts)
    return {"shape": SHAPE_SORT, "key_mode": mode, "sort_on_key8": int(key8), "destroy_threshold": 0,
            "seed": seed, "init_counts": counts, "creates": [0] * W, "kill_steps": [0] * W}


def _counts_for(n):
    """Worlds and per-world counts for a custom-key table of n rows."""
    rng = np.random.default_rng(n)
    if n == 1:
        return [1]
    if n <= 2049:
        return _uneven(n, 5, rng, empty_every=3)
    if n <= 20_000:
        return _uneven(n, 9, rng, empty_every=4)
    if n <= 200_000:
        counts = _uneven(n - 30_000, 99, rng, empty_every=5)
        return counts[:7] + [30_000] + counts[7:]         # one world spanning ~15 tiles
    return _uneven(n, 96, rng, empty_every=5)


ROWS = [1, 2047, 2048, 2049, 9 * TILE + 1, 64 * TILE + 5, 1_200_003]


@pytest.mark.gpu
@pytest.mark.parametrize("n", ROWS)
@pytest.mark.parametrize("key8", [False, True], ids=["key4", "key8"])
def test_custom_key_sort_uniform_keys(n, key8, monkeypatch):
    # one key in 16 is 0xFFFFFFFF and must be kept, not truncated
    if n > 1_000_000:
        # a growable table reserves 64x its initial rows: start the 96 worlds with 1024 each
        monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "1024")
    _run_case(_sort_cfg(_counts_for(n), KEY_UNIFORM, key8), steps=3, expect_rows=n)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2049, 64 * TILE + 5])
@pytest.mark.parametrize("mode", [KEY_CONSTANT, KEY_ALL_ONES, KEY_BYTE3], ids=["constant", "all_ones", "byte3"])
@pytest.mark.parametrize("key8", [False, True], ids=["key4", "key8"])
def test_custom_key_sort_key_distributions(n, mode, key8):
    # constant / all-ones keys put every row in one digit (look-back sums reach n); byte-3 keys
    # are decided by the last of the four passes alone
    _run_case(_sort_cfg(_counts_for(n), mode, key8), steps=3, expect_rows=n)


def _churn_cfg(W, seed=5, steps_kill=None):
    rng = np.random.default_rng(W)
    if W == 1:
        init, creates = [20_000], [300]
    else:
        init = [int(x) for x in rng.integers(1, 7, W)]
        creates = [int(x) for x in rng.integers(0, 3, W)]
        for w in range(0, W, 5):            # every 5th world stays empty
            init[w] = creates[w] = 0
    kill = [2 if w % 7 == 3 else 0 for w in range(W)] if steps_kill is None else [steps_kill] * W
    if W > 1 and steps_kill is None:
        # the last world holds rows at every step: its ID is the one whose low digits equal a
        # destroyed row's all-ones key when the world sort runs one radix pass too few
        init[W - 1], creates[W - 1], kill[W - 1] = max(init[W - 1], 3), max(creates[W - 1], 1), 0
    return {"shape": SHAPE_CHURN, "key_mode": KEY_UNIFORM, "sort_on_key8": 0, "seed": seed,
            "destroy_threshold": int(0.2 * 2 ** 32), "init_counts": init, "creates": creates, "kill_steps": kill}


@pytest.mark.gpu
@pytest.mark.parametrize("W", [1, 255, 256, 257, 65535, 65536, 65537])
def test_world_sort_with_churn(W, monkeypatch):
    # 255 -> 256 and 65535 -> 65536 worlds add a radix pass; world W - 1 always has rows (one pass
    # too few would mix them with destroyed rows); other worlds w % 7 == 3 delete every row at step 2
    assert restate.world_sort_passes(W) == (1 if W < 256 else 2 if W < 65536 else 3)
    if W == 1:
        monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "1024")    # the single world's 20 000 rows
    _run_case(_churn_cfg(W), steps=4)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [3, 300])
def test_step_deleting_every_row(W):
    # every world deletes all of its rows at step 2 and makes none: the table empties, then refills
    cfg = _churn_cfg(W, steps_kill=2)
    cfg["init_counts"] = [max(c, 1) for c in cfg["init_counts"]]
    cfg["creates"] = [max(c, 1) for c in cfg["creates"]]
    model = Model(cfg)
    model.step()
    model.step()
    assert model.n == 0
    assert _run_case(cfg, steps=4).n > 0


@pytest.mark.gpu
@pytest.mark.parametrize("key8,mode", [(False, KEY_UNIFORM), (True, KEY_BYTE3), (False, KEY_CONSTANT)],
                         ids=["key4_uniform", "key8_byte3", "key4_constant"])
def test_custom_sort_over_destroyed_rows_then_compaction(key8, mode):
    cfg = _churn_cfg(257)
    cfg.update(shape=SHAPE_REKEY_CHURN_SORT, key_mode=mode, sort_on_key8=int(key8))
    cfg["init_counts"][1] = 5000           # one world over two tiles
    _run_case(cfg, steps=4)


@pytest.mark.gpu
def test_custom_sort_marks_table_for_the_next_world_sort():
    # no churn: only the custom sort's needsSort makes the compaction regroup the rows by world
    W = 40
    counts = _uneven(3000, W, np.random.default_rng(3), empty_every=6)
    cfg = {"shape": SHAPE_REKEY_CHURN_SORT, "key_mode": KEY_UNIFORM, "sort_on_key8": 0, "seed": 9,
           "destroy_threshold": 0, "init_counts": counts, "creates": [0] * W, "kill_steps": [0] * W}
    _run_case(cfg, steps=3, expect_rows=3000)


@pytest.mark.gpu
def test_tables_and_sort_scratch_grow_between_steps(monkeypatch):
    # 2 rows per world to start with (256 rows): the table, its twin buffers and the sort
    # scratch must grow between steps (twice at least: ~650 live rows at the end) while
    # exported pointers stay put
    monkeypatch.setenv("MADRONA_B200_ROWS_PER_WORLD", "2")
    W = 100
    cfg = {"shape": SHAPE_REKEY_CHURN_SORT, "key_mode": KEY_UNIFORM, "sort_on_key8": 1, "seed": 2,
           "destroy_threshold": int(0.1 * 2 ** 32), "init_counts": [1] * W,
           "creates": [1] * W, "kill_steps": [0] * W}
    model = _run_case(cfg, steps=9)
    assert model.n > 2 * 256
