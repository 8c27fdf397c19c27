"""-m gpu: randomized differential test — random schemas (sizes, optional columns, byte-range checksums), random
compiled systems, random populations, random VALID request vectors (plain ticks, rollbacks of random depth into the
snapshots that exist, spectator-style catch-up runs), random host edits between vectors (remove / insert of optional
components, spawns), and the occasional invalid rollback.  After every vector: checksums, frame resources and ring
contents equal the oracle's; periodically every column, presence bit and the alive set.  Each seed runs on the default
one-launch path and on the stepwise path.  A second schema generator reaches the wide rows and long checksum ranges
that pick other kernels: rows too wide for the NVRTC kernel (> 24 words), for the one-launch program and two TMA stages
(> 49 words), a 1024-byte element, ranges up to the element's end, 6 checksummed and 7 optional columns, 8 and 9
systems."""
import numpy as np
import pytest

from bevy_ggrs_b200 import capi
from bevy_ggrs_b200.capi import BgrError
from bevy_ggrs_b200.engine import Engine
from bevy_ggrs_b200.session import ADVANCE, LOAD, SAVE, Request
from oracle_backend import OracleError, OracleWorld
from schema_util import WIDE_PATHS, expected_kind as _expected_kind, path_env as _path_env

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300), pytest.mark.usefixtures("generic_kernel")]
NOSESS = (capi.BGR_SESSION_NONE, 0, 0, 0)
OPT = capi.BGR_STRATEGY_OPTIONAL


def _make_worlds(rng, flags):
    n = int(rng.integers(1, 1400))
    depth = int(rng.integers(2, 9))
    n_cols = int(rng.integers(1, 5))
    sizes = [int(rng.choice([1, 4, 4, 8, 12, 16, 40, 7])) for _ in range(n_cols)]
    optional = [bool(rng.random() < 0.5) for _ in range(n_cols)]
    worlds = [Engine(max_entities=n + 64, max_depth=depth + 1, flags=flags), OracleWorld()]
    cols = []
    for w in worlds:
        cols = [w.rollback_component(f"C{i}", sizes[i], (capi.BGR_STRATEGY_COPY | OPT) if optional[i] else capi.BGR_STRATEGY_CLONE)
                for i in range(n_cols)]
    # checksums: random byte ranges (aligned and unaligned)
    cks = []
    for i in range(n_cols):
        if rng.random() < 0.7:
            off = int(rng.integers(0, sizes[i]))
            ln = int(rng.integers(1, sizes[i] - off + 1))
            if rng.random() < 0.5 and sizes[i] >= 4:
                off, ln = 0, sizes[i] - sizes[i] % 4
            cks.append((i, off, max(1, ln)))
    for w in worlds:
        for i, off, ln in cks:
            w.checksum_component(cols[i], off, ln)
    # systems on columns that have a u32 field
    systems = []
    for i in range(n_cols):
        if sizes[i] >= 4 and sizes[i] % 4 == 0 and rng.random() < 0.8:
            off = 4 * int(rng.integers(0, sizes[i] // 4))
            kind = rng.choice([capi.BGR_SYS_U32_ADD, capi.BGR_SYS_U32_SATSUB_DESPAWN, capi.BGR_SYS_U32_STORE_CALL_COUNT])
            if kind == capi.BGR_SYS_U32_STORE_CALL_COUNT:
                systems.append((int(kind), [cols[i]], [off]))
            else:
                systems.append((int(kind), [cols[i]], [off, int(rng.integers(1, 4))]))
    if optional and rng.random() < 0.5:
        i = int(rng.integers(0, n_cols))
        systems.append((capi.BGR_SYS_DESPAWN_ON_INPUT, [cols[i]], [0, 3]))
    for w in worlds:
        for sid, c, p in systems:
            w.add_system(sid, c, p)
        w.build()
        w.set_depth(depth)
    data = [rng.integers(0, 256, (n, sizes[i]), dtype=np.uint8) for i in range(n_cols)]
    for i in range(n_cols):   # u32 fields small enough that SATSUB despawns some entities inside the run
        if sizes[i] % 4 == 0:
            data[i].view(np.uint32)[:] = rng.integers(1, 30, (n, sizes[i] // 4), dtype=np.uint32)
    removes = [(i, int(r)) for i in range(n_cols) if optional[i] for r in rng.choice(n, size=min(n, int(rng.integers(0, 20))), replace=False)]
    for w in worlds:
        w.spawn(n)
        for i in range(n_cols):
            w.write_component(cols[i], 0, data[i])
        for i, r in removes:
            w.remove_component(cols[i], r)
    return worlds[0], worlds[1], cols, sizes, optional, depth


def _compare_state(eng, orc, cols):
    rows = eng.row_count()
    assert rows == orc.row_count()
    alive = orc.read_alive(0, rows).astype(bool)
    assert np.array_equal(eng.read_alive(0, rows).astype(bool), alive)
    for c in cols:
        vo, ho = orc.read_component_alive(c, 0, rows)
        he = eng.has_component(c, 0, rows).astype(bool)
        assert np.array_equal(he, ho.astype(bool)), f"presence of column {c}"
        assert np.array_equal(eng.read_component(c, 0, rows)[he], vo[he]), f"values of column {c}"


def _drive(eng, orc, cols, sizes, optional, rng, flags, seed, n_vectors=40, input_hi=5, insert_value=None, allow_host_spawn=True,
           expect_kind=None):
    frame = 0  # RollbackFrameCount of both worlds
    for step in range(n_vectors):
        frames = orc.snapshot_frames()
        assert eng.snapshot_frames() == frames
        choice = rng.random()
        reqs = []
        inp = lambda: [int(rng.integers(0, input_hi))]
        if choice < 0.45 or not frames:                       # a plain tick
            reqs = [Request(SAVE, frame), Request(ADVANCE, 0, inp())]
            frame += 1
        elif choice < 0.85:                                   # a rollback into a snapshot that exists, then resimulation
            g = int(rng.choice(frames))
            reqs = [Request(LOAD, g)]
            f = g
            for k in range(frame - g):
                if k > 0:
                    reqs.append(Request(SAVE, f))
                reqs.append(Request(ADVANCE, 0, inp()))
                f += 1
            reqs += [Request(SAVE, f), Request(ADVANCE, 0, inp())]
            frame = f + 1
        else:                                                 # spectator-style catch-up: advances only
            k = int(rng.integers(1, 4))
            reqs = [Request(ADVANCE, 0, inp()) for _ in range(k)]
            frame += k
        a, b = eng.handle_requests(NOSESS, reqs), orc.handle_requests(NOSESS, reqs)
        assert a == b, f"seed {seed} step {step}"
        assert eng.rollback_frame_count() == orc.rollback_frame_count() == frame
        if expect_kind is not None:
            assert eng.last_kernel().kind == expect_kind, f"seed {seed} step {step}"
        elif flags == 0:
            assert eng.last_path_fused()
        # host edits between vectors
        rows = orc.row_count()
        alive = np.flatnonzero(orc.read_alive(0, rows))
        opt_cols = [i for i, o in enumerate(optional) if o]
        if opt_cols and alive.size and rng.random() < 0.5:
            for r in rng.choice(alive, size=min(3, alive.size), replace=False):
                i = int(rng.choice(opt_cols))
                if orc.has_component(cols[i], int(r), 1)[0]:
                    for w in (eng, orc):
                        w.remove_component(cols[i], int(r))
                else:
                    val = insert_value(i, rng) if insert_value else rng.integers(1, 200, sizes[i], dtype=np.uint8)
                    for w in (eng, orc):
                        w.insert_component(cols[i], int(r), val)
        if allow_host_spawn and rng.random() < 0.1 and rows < eng.max_entities - 8:
            k = int(rng.integers(1, 6))
            vals = [rng.integers(1, 40, (k, s), dtype=np.uint8) for s in sizes]
            for w in (eng, orc):
                first = w.spawn(k)
                for i, c in enumerate(cols):
                    w.write_component(c, first, vals[i])
        if step % 8 == 7:
            _compare_state(eng, orc, cols)
    _compare_state(eng, orc, cols)
    # Last: an invalid rollback.  The reference panics ("Could not rollback to ...", mod.rs:209-212) after popping every
    # snapshot on its way — the app is dead at that point, so nothing after it is compared; the engine reports the same
    # text as a status and has executed nothing (its ring is untouched).
    before = eng.snapshot_frames()
    with pytest.raises(BgrError) as ee:
        eng.handle_requests(NOSESS, [Request(LOAD, frame + 1000)])
    with pytest.raises(OracleError) as eo:
        orc.handle_requests(NOSESS, [Request(LOAD, frame + 1000)])
    assert ee.value.status == capi.BGR_ERR_NO_SNAPSHOT and str(ee.value) == str(eo.value)
    assert eng.snapshot_frames() == before and eng.rollback_frame_count() == frame


@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
@pytest.mark.parametrize("seed", list(range(12)))
def test_random_worlds_and_request_vectors_match_the_oracle(seed, flags):
    rng = np.random.default_rng(1000 + seed)
    eng, orc, cols, sizes, optional, depth = _make_worlds(rng, flags)
    _drive(eng, orc, cols, sizes, optional, rng, flags, seed)
    eng.close(); orc.close()


@pytest.mark.parametrize("flags", [0, capi.BGR_CFG_FORCE_STEPWISE])
@pytest.mark.parametrize("seed", list(range(8)))
def test_random_request_vectors_on_the_particles_bundle_match_the_oracle(seed, flags):
    """The stress-test bundle under the same random driver: random optional flags on Velocity / Ttl (fused kernel MODE 2),
    an optional extra passive column of odd size, spawn_particles on random inputs (INPUT_SPAWN = 1 << 4) when no column
    is optional, particles dying inside the window, random rollbacks / catch-up runs / invalid rollbacks."""
    from bevy_ggrs_b200.stress import synth_particles
    rng = np.random.default_rng(5000 + seed)
    n = int(rng.integers(1, 3000))
    depth = int(rng.integers(2, 9))
    opt_v, opt_l = bool(rng.random() < 0.4), bool(rng.random() < 0.4)
    extra = int(rng.choice([0, 0, 5, 16]))
    spawn = (not opt_v and not opt_l) and rng.random() < 0.6
    rate = int(rng.integers(1, 40))
    worlds = [Engine(max_entities=n + 20000, max_depth=depth + 1, flags=flags), OracleWorld()]   # room for every possible spawn
    for w in worlds:
        t = w.rollback_component("Transform", 40, capi.BGR_STRATEGY_CLONE)
        v = w.rollback_component("Velocity", 12, capi.BGR_STRATEGY_COPY | (OPT if opt_v else 0))
        l = w.rollback_component("Ttl", 8, capi.BGR_STRATEGY_COPY | (OPT if opt_l else 0))
        cols, sizes, optional = [t, v, l], [40, 12, 8], [False, opt_v, opt_l]
        if extra:
            cols.append(w.rollback_component("Extra", extra, capi.BGR_STRATEGY_COPY)); sizes.append(extra); optional.append(False)
        w.checksum_component(v, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)
        w.checksum_component(t, 0, 12, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)
        if spawn:
            w.add_system(capi.BGR_SYS_PARTICLES_SPAWN, [t, v, l], [rate, 6, 123, 0])
        w.add_system(capi.BGR_SYS_PARTICLES_UPDATE, [t, v])
        w.add_system(capi.BGR_SYS_PARTICLES_DESPAWN, [l])
        w.build()
        w.set_depth(depth)
        tf, vel, ttl = synth_particles(n, 900 + seed, 2, 25, z_fraction=0.3)
        w.spawn(n)
        w.write_component(t, 0, tf); w.write_component(v, 0, vel); w.write_component(l, 0, ttl)
        if extra:
            w.write_component(cols[3], 0, np.random.default_rng(seed).integers(0, 256, (n, extra), dtype=np.uint8))
    eng, orc = worlds

    def insert_value(i, r):
        if i == 1:
            return np.array([1.5, -2.5, 0.25], np.float32).view(np.uint8)
        return np.array([int(r.integers(2, 20))], np.uint64).view(np.uint8)
    _drive(eng, orc, cols, sizes, optional, rng, flags, seed, n_vectors=32, input_hi=32, insert_value=insert_value, allow_host_spawn=False)
    eng.close(); orc.close()


# ---------------------------------------------------------------------------------------------------------------------
# wide rows and long checksum ranges
# ---------------------------------------------------------------------------------------------------------------------
WIDE_WORDS = [24, 25, 49, 50, 256]   # 256: one 1024-byte element
RANGE_LENS = [0, 1, 3, 4, 8, 12, 16, 20, 31, 32, 33, 60, 64, 68]
U32_SYSTEMS = [capi.BGR_SYS_U32_ADD, capi.BGR_SYS_U32_SATSUB_DESPAWN, capi.BGR_SYS_U32_STORE_CALL_COUNT]


def _make_wide_worlds(rng, flags, words, aligned):
    """Columns that add up to `words` words (sub-word tails included), up to 7 optional, up to 6 checksummed over
    ranges of the lengths and offsets that change code paths, and 2, 8 or 9 u32 systems."""
    n = int(rng.integers(1, 1400))
    depth = int(rng.integers(2, 9))
    if words == 256:
        col_words = [256]
    else:
        n_cols = int(rng.integers(2, 9))
        cuts = sorted(rng.choice(np.arange(1, words), size=n_cols - 1, replace=False).tolist())
        col_words = [b - a for a, b in zip([0] + cuts, cuts + [words])]
    sizes = [4 * w - (int(rng.integers(0, 4)) if (rng.random() < 0.3 and not aligned) else 0) for w in col_words]
    n_opt = min(len(sizes), int(rng.choice([0, 2, 7])))
    optional = [i < n_opt for i in range(len(sizes))]
    rng.shuffle(optional)
    worlds = [Engine(max_entities=n + 64, max_depth=depth + 1, flags=flags), OracleWorld()]
    cols = []
    for w in worlds:
        cols = [w.rollback_component(f"W{i}", sizes[i], (capi.BGR_STRATEGY_COPY | OPT) if optional[i] else capi.BGR_STRATEGY_CLONE)
                for i in range(len(sizes))]
    cks, nvrtc_ranges = [], True
    for i in rng.permutation(len(sizes))[:6]:
        size = sizes[i]
        if aligned:   # whole words, 4..64 bytes: the ranges the NVRTC kernel accepts (lanes wrap past 32 bytes)
            ln = min(int(rng.choice([4, 8, 12, 16, 20, 32, 60, 64])), size - size % 4)
            off = 4 * int(rng.integers(0, (size - ln) // 4 + 1))
        else:
            off = int(rng.choice([0, 1, 2, 3, 4 * int(rng.integers(0, max(1, size // 4)))]))
            off = min(off, size)
            ln = int(rng.choice(RANGE_LENS + [size - off]))
            ln = min(ln, size - off)
        nvrtc_ranges = nvrtc_ranges and (off % 4 == 0 and ln % 4 == 0 and 4 <= ln <= 64)
        cks.append((int(i), off, ln))
    for w in worlds:
        for i, off, ln in cks:
            w.checksum_component(cols[i], off, ln)
    u32_cols = [i for i in range(len(sizes)) if sizes[i] >= 4]
    systems = []
    for _ in range(int(rng.choice([2, 8, 9]))):
        i = int(rng.choice(u32_cols))
        off = 4 * int(rng.integers(0, sizes[i] // 4))
        kind = int(rng.choice(U32_SYSTEMS))
        systems.append((kind, [cols[i]], [off] if kind == capi.BGR_SYS_U32_STORE_CALL_COUNT else [off, int(rng.integers(1, 4))]))
    for w in worlds:
        for sid, c, p in systems:
            w.add_system(sid, c, p)
        w.build()
        w.set_depth(depth)
    data = [rng.integers(0, 256, (n, s), dtype=np.uint8) for s in sizes]
    for i, s in enumerate(sizes):   # small u32 words: SATSUB despawns inside the run
        if s % 4 == 0:
            data[i].view(np.uint32)[:] = rng.integers(1, 30, (n, s // 4), dtype=np.uint32)
    removes = [(i, int(r)) for i in range(len(sizes)) if optional[i] for r in rng.choice(n, size=min(n, 6), replace=False)]
    for w in worlds:
        w.spawn(n)
        for i in range(len(sizes)):
            w.write_component(cols[i], 0, data[i])
        for i, r in removes:
            w.remove_component(cols[i], r)
    return worlds[0], worlds[1], cols, sizes, optional, len(systems), nvrtc_ranges


@pytest.mark.parametrize("path", list(WIDE_PATHS))
@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("words", WIDE_WORDS)
def test_wide_rows_and_long_ranges_match_the_oracle(monkeypatch, generic_kernel, words, seed, path):
    flags = _path_env(monkeypatch, path, generic_kernel)
    rng = np.random.default_rng(9000 + 17 * words + seed)
    aligned = seed == 0 and words <= 24    # seed 0 of the narrow class stays inside what the NVRTC kernel accepts
    eng, orc, cols, sizes, optional, n_sys, nvrtc_ranges = _make_wide_worlds(rng, flags, words, aligned)
    kind = _expected_kind(path, words, n_sys, nvrtc_ranges, generic_kernel)
    _drive(eng, orc, cols, sizes, optional, rng, flags, seed, n_vectors=24, expect_kind=kind)
    eng.close(); orc.close()


@pytest.mark.parametrize("path", ["generic", "stepwise_tma", "stepwise_flat"])
@pytest.mark.parametrize("elem,off,ln", [(96, 4, 64), (196, 8, 188), (1024, 0, 1024), (1024, 512, 508)])
def test_finite_assertion_covers_the_whole_long_range(monkeypatch, generic_kernel, elem, off, ln, path):
    """A finite-checked range that ends inside the element: inf in its last word raises BGR_ERR_NON_FINITE (the oracle
    panics), inf in the word right after it does not.  Every kernel that hashes such a range: the one-launch program
    (interpreter; NVRTC up to 64 bytes), the TMA copy kernel and k_checksum_column."""
    flags = _path_env(monkeypatch, path, generic_kernel)
    words = elem // 4
    kind = _expected_kind(path, words, 0, ln <= 64, generic_kernel)
    for word, raises in ((off + ln) // 4 - 1, True), ((off + ln) // 4, False):
        if word >= words:
            continue
        eng, orc = Engine(max_entities=1200, max_depth=4, flags=flags), OracleWorld()
        data = np.random.default_rng(elem + word).uniform(-9.0, 9.0, (1100, words)).astype(np.float32)
        data[1037, word] = np.inf
        res = []
        for w in (eng, orc):
            c = w.rollback_component("Wide", elem, capi.BGR_STRATEGY_COPY)
            w.checksum_component(c, off, ln, capi.BGR_HASH_FLAG_ASSERT_FINITE_F32)
            w.build()
            w.spawn(1100)
            w.write_component(c, 0, data)
            try:
                res.append(("ok", w.handle_requests(NOSESS, [Request(SAVE, 0), Request(ADVANCE, 0, [0]), Request(SAVE, 1)])))
            except (BgrError, OracleError) as ex:
                res.append(("raised", ex.status, str(ex)))
        assert res[0] == res[1]
        assert res[0][0] == ("raised" if raises else "ok")
        if raises:
            assert res[0][1] == capi.BGR_ERR_NON_FINITE
        assert eng.last_kernel().kind == kind
        eng.close(); orc.close()


def test_a_1024_byte_column_round_trips(generic_kernel):
    """write_component -> read_component (whole and a sub-range) and peek of a saved frame for a 1024-byte element
    (256 word planes) next to a 3-byte one."""
    n = 700
    eng = Engine(max_entities=n, max_depth=4)
    c = eng.rollback_component("Blob", 1024, capi.BGR_STRATEGY_CLONE)
    small = eng.rollback_component("Small", 3, capi.BGR_STRATEGY_COPY)
    eng.checksum_component(c, 0, 1024)
    eng.build()
    eng.spawn(n)
    data = np.random.default_rng(5).integers(0, 256, (n, 1024), dtype=np.uint8)
    eng.write_component(c, 0, data)
    eng.write_component(small, 0, data[:, :3])
    assert np.array_equal(eng.read_component(c, 0, n), data)
    assert np.array_equal(eng.read_component(c, 300, 17), data[300:317])
    eng.handle_requests(NOSESS, [Request(SAVE, 0)])
    assert eng.last_kernel().kind == "stepwise_flat"
    eng.write_component(c, 0, data[::-1].copy())
    pe = eng.peek(0, c, 0, n)
    assert pe is not None and pe[1].all() and np.array_equal(pe[0], data)
    assert np.array_equal(eng.read_component(c, 0, n), data[::-1])
    eng.close()
