"""Deferred common ages (DESIGN.md §3) on the real hnb_init / hnb_update kernels under the CPU thread emulation, with
BatchParams::defer_ages set as the runtime sets it for the authored C5: a floor group whose 32 rows all survive keeps its age
in its word and its age column is not stored; an update that meets the group outside a floor tile takes the age from the
word, and the 32nd row to do so ends the deferral; k_flush_group_ages writes deferred ages back for every other reader or
writer of records.

Each frame is compared with the oracle through the records with every deferred age put back (`materialised`), so the
deferrals carry over from frame to frame as on the device. Every test runs at K = 1, 2, 4 and 8 rows in flight per lane
(HNB_TILE_K), with 1, 2 and the most sub-tiles a tile holds."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from bevy_hanabi_b200 import recipes
from tests import static_emu as S
from tests.effects import ROWS_PER_LANE
from tests.helpers import Instance
from tests.kernel_emu import CLAIMED_DRIVER, EmuWorld, assert_same, c5_frame, c5_world, claim

pytestmark = pytest.mark.timeout(900)

NONE = np.uint32(0xFFFFFFFF)
WORD_NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
RO_REAP = 1 | 2  # HNB_ATTR_UPDATE_READ_ONLY | HNB_ATTR_REAP_ONLY
SHAPES = [(k, n) for k in (1, 2, 4, 8) for n in sorted({1, 2, ROWS_PER_LANE // k})]
TILE_SHAPES = pytest.mark.parametrize("k,chunks", SHAPES, ids=[f"K{k}-{n}sub" for k, n in SHAPES])
AGE_WORD = 3
AGE_COL = 2  # column [24, 28) of the C5 word map holds the age alone


@pytest.fixture(autouse=True)
def _default_shape(monkeypatch):
    for v in ("HNB_TILE_K", "HNB_ROWS_PER_LANE", "HNB_DEFINES"):
        monkeypatch.delenv(v, raising=False)


# The emulation driver with identity claims whose launches pass the slab's floors and common ages, with deferral on.
_PARAMS = """static hnb::BatchParams make_params(const EmuBatch* b) {
    hnb::BatchParams P;
    memset((void*)&P, 0, sizeof(P));
"""
assert CLAIMED_DRIVER.count(_PARAMS) == 1
DEFER_DRIVER = CLAIMED_DRIVER.replace(_PARAMS, """static float* g_life_floor = nullptr;
static unsigned long long* g_group_age = nullptr;
extern "C" void emu_set_group_words(float* floors, unsigned long long* ages) { g_life_floor = floors; g_group_age = ages; }
""" + _PARAMS + """    P.life_floor = g_life_floor;
    P.group_age = g_group_age;
    P.defer_ages = 1u;
""")

FLUSH_DRIVER = r"""
extern "C" void semu_flush_group_ages(const PlaneSet* ps, uint32_t age_word, unsigned long long* ages, uint32_t* floors, uint32_t first,
                                      uint32_t count, uint32_t capacity, uint32_t clear, uint32_t epoch) {
    const PlaneSet p = *ps;
    if (count == 0) return;
    const uint32_t g0 = first >> 5, groups = uint32_t(((uint64_t(first) + count + 31u) >> 5) - g0);  // as launch_flush_group_ages
    emu_run([&] { k_flush_group_ages(p, age_word, ages, floors, g0, groups, capacity, clear, epoch); }, (groups + 255u) / 256u, 256);
}
"""
_FLUSH_LIB = []


def flush_lib():
    if not _FLUSH_LIB:
        lib = S.build(FLUSH_DRIVER)
        lib.semu_flush_group_ages.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p] + [C.c_uint32] * 5
        lib.semu_flush_group_ages.restype = None
        _FLUSH_LIB.append(lib)
    return _FLUSH_LIB[0]


def c5_with_floors():
    fx = recipes.c5_lowered()
    return dataclasses.replace(fx, attrs=[dataclasses.replace(a, flags=RO_REAP if a.name == "lifetime" else 0) for a in fx.attrs])


def plane_set(planes, columns):
    """hnb::PlaneSet of 1-D column arrays (row-major, len(words) u32 per row) holding the record words `columns`."""
    ps = S.PlaneSet()
    for p, words in enumerate(columns):
        ps.ptr[p] = planes[p].ctypes.data
        ps.words[p] = len(words)
        ps.word_off[p] = words[0] if words == list(range(words[0], words[0] + len(words))) else \
            0x80000000 | sum(w << (6 * l) for l, w in enumerate(words))
        for w in words:
            ps.word_to_plane[w] = p
    return ps


class World:
    def __init__(self, n, cap, chunks, k, monkeypatch, lifetimes=None, ages=None, seed=1):
        monkeypatch.setenv("HNB_TILE_K", str(k))
        self.ref = c5_world(np.random.default_rng(seed), [Instance(0, cap, alive=n, seed=42)])
        self.ref.particles[:n, 7] = np.asarray(lifetimes if lifetimes is not None else np.full(n, 5.0), dtype=np.float32).view(np.uint32)
        if ages is not None:
            self.ref.particles[:n, 3] = np.asarray(ages, dtype=np.float32).view(np.uint32)
        fx = c5_with_floors()
        src = fx.generate_source()
        assert f"#define HNB_GROUP_AGE_WORD {AGE_WORD}\n" in src and "hnb_store_written_but_age" in src and "hnb_store_age" in src
        self.columns = fx.column_words()
        assert self.columns[AGE_COL] == [AGE_WORD]
        self.emu = emu = EmuWorld(self.ref, fx, chunks=chunks, update_ctas=2, driver=DEFER_DRIVER)
        assert emu.lib.emu_tile_k() == k and emu.tile == 32 * k * chunks
        self.claims = np.array([claim(0, n)] * 2, dtype=np.uint64)
        emu.lib.emu_set_ident_claim.argtypes = [C.c_void_p]
        emu.lib.emu_set_ident_claim.restype = None
        emu.lib.emu_set_ident_claim(self.claims.ctypes.data)
        self.floors = np.full(cap // 32 + 1, NONE, dtype=np.uint32)
        self.words = np.full(cap // 32 + 2, WORD_NONE, dtype=np.uint64)  # the groups' words, then the count of deferred ones
        self.words[-1] = 0
        emu.lib.emu_set_group_words.argtypes = [C.c_void_p, C.c_void_p]
        emu.lib.emu_set_group_words.restype = None
        emu.lib.emu_set_group_words(self.floors.ctypes.data, self.words.ctypes.data)
        self.cap = cap

    def frame(self, orc, spawn=0):
        c5_frame(orc, self.ref, self.emu, spawn)

    def deferred(self):
        return (self.words[:-1] >> np.uint64(62)) == 1

    def materialised(self):
        """What the emulated slab holds with every deferred age written back (the update's state left as it is)."""
        got = self.emu.pull()
        for g in np.nonzero(self.deferred())[0]:
            got["particles"][g * 32:(g + 1) * 32, AGE_WORD] = np.uint32(int(self.words[g]) & 0xFFFFFFFF)
        return got

    def check(self, what):
        assert_same(self.ref, self.materialised(), what)
        # after a launch every deferred word is a floor tile's (no row counted), and no other word has the deferred bits
        d = self.deferred()
        assert ((self.words[:-1][d] >> np.uint64(32)) == np.uint64(1 << 30)).all(), f"{what}: a deferred word with rows counted"
        assert int(self.words[-1]) == int(d.sum()), f"{what}: the count of deferred words"
        return d

    def flush(self, first, count, clear, epoch=0):
        ps = plane_set(self.emu.planes, self.columns)
        flush_lib().semu_flush_group_ages(C.byref(ps), AGE_WORD, self.words.ctypes.data, self.floors.ctypes.data, first, count, self.cap,
                                          int(clear), epoch)


def _floor_groups(emu, n):
    return (n // emu.tile) * emu.tile // 32


@TILE_SHAPES
def test_steady_state_defers_and_stores_no_age(orc, monkeypatch, k, chunks):
    """Frame 0 loads the fill's ages and defers every floor group. The age column is then poisoned under them: the update
    neither reads nor writes it, each frame's words carry the oracle's ages, and the flush puts the oracle's records back."""
    n, cap = 2900, 3200
    w = World(n, cap, chunks, k, monkeypatch)
    full = _floor_groups(w.emu, n)
    assert full > 0
    w.frame(orc)
    d = w.check("frame 0")
    assert d[:full].all() and not d[full:].any()
    np.testing.assert_array_equal((w.words[:full] & np.uint64(0xFFFFFFFF)).astype(np.uint32),
                                  np.full(full, np.float32(w.ref.sim.delta_time)).view(np.uint32))
    col = w.emu.planes[AGE_COL]
    col[:full * 32] = np.uint32(0x7FC0DEAD)
    for step in range(1, 4):
        w.frame(orc)
        assert w.check(f"frame {step}")[:full].all()
        assert (col[:full * 32] == np.uint32(0x7FC0DEAD)).all(), "the update stored ages of deferred groups"
    w.flush(0, cap, clear=False, epoch=w.emu.epoch)
    assert_same(w.ref, w.emu.pull(), "after the flush")
    assert (w.words[:full] >> np.uint64(32) == np.uint64(w.emu.epoch)).all(), "a reader's flush leaves known words"
    for step in range(4, 6):  # known words are read as such, and the groups are deferred again
        w.frame(orc)
        assert w.check(f"frame {step}")[:full].all()


@TILE_SHAPES
def test_deaths_in_deferred_groups_then_spawns(orc, monkeypatch, k, chunks):
    """Rows of deferred groups die (a whole group, and single rows of others): those groups store their ages and leave
    words that are not deferred, the list becomes a gather so that later deferred groups are consumed outside floor tiles,
    and the next frames spawn into the freed slots."""
    n, cap = 2048, 2048
    life = np.full(n, 5.0, dtype=np.float32)
    life[96:128] = 0.05          # group 3 dies whole
    life[[5, 300, 1000]] = 0.07  # single rows of groups 0, 9, 31
    w = World(n, cap, chunks, k, monkeypatch, lifetimes=life, seed=4)
    for step in range(8):
        w.frame(orc, spawn=40 if step in (5, 6) else 0)
        w.check(f"frame {step}")
    w.flush(0, cap, clear=True)
    assert_same(w.ref, w.emu.pull(), "after a writer's flush")
    assert (w.words[:-1] == WORD_NONE).all() and (w.floors == NONE).all() and w.words[-1] == 0


@pytest.mark.parametrize("k", [1, 2, 4, 8], ids=lambda k: f"K{k}")
def test_tile_size_changes_and_split_groups(orc, monkeypatch, k):
    """The tile size changes from frame to frame under a claim that ends inside a tile, so deferred groups reach tiles that
    are not floor tiles; after one death near the front every later group is split between two rows of 32 list entries,
    i.e. two warps (and, with one sub-tile of K = 1, two tiles). Every deferred word consumed outside a floor tile is the
    sentinel after the launch, and its 32 rows hold its age plus dt."""
    n, cap = 1000, 4096
    life = np.full(n, 5.0, dtype=np.float32)
    life[3] = 0.04
    w = World(n, cap, 1, k, monkeypatch, lifetimes=life, seed=5)
    most = ROWS_PER_LANE // k
    chunk_seq = [c for c in (1, most, 2, most, 1, 3, most, 2, 1, most) if c <= most]
    outside = 0
    for f, chunks in enumerate(chunk_seq):
        emu = w.emu
        emu.tile_word = emu.b.tile_rows = emu.tile = 32 * k * chunks
        before = w.deferred().copy()
        w.frame(orc)
        d = w.check(f"frame {f}, {chunks} sub-tiles")
        # a floor tile that takes a deferred word and does not defer it again leaves it known (or the sentinel); outside
        # floor tiles the 32nd row leaves the sentinel
        consumed = w.words[:-1][before & ~d]
        assert ((consumed == WORD_NONE) | ((consumed >> np.uint64(32)) == np.uint64(emu.epoch))).all()
        outside += int((consumed == WORD_NONE).sum())
    assert outside > 0, "no deferred group reached a tile that is not a floor tile"


@pytest.mark.parametrize("k", [1, 4], ids=lambda k: f"K{k}")
def test_batch_sits_out_while_deferred(orc, monkeypatch, k):
    """Frames in which the batch is not launched advance the epoch only: a deferred word needs no epoch test."""
    n, cap = 2048, 2048
    w = World(n, cap, 2, k, monkeypatch)
    for gap in (1, 3, 70):
        w.frame(orc)
        assert w.check(f"before a gap of {gap}").any()
        w.emu.epoch += gap
        w.frame(orc)
        w.check(f"after a gap of {gap}")


@TILE_SHAPES
def test_special_values(orc, monkeypatch, k, chunks):
    """Groups with one differing age, all-ones ages, -0.0, NaN and infinite lifetimes and common negative ages, and frames
    with dt = 0: nothing of that defers a group it must not, and every frame matches the oracle."""
    n, cap = 2048, 2048
    rng = np.random.default_rng(9)
    life = rng.uniform(0.2, 2.0, n).astype(np.float32)
    life[rng.choice(n, 12, replace=False)] = np.nan
    life[rng.choice(n, 12, replace=False)] = np.inf
    life[rng.choice(n, 12, replace=False)] = -np.inf
    ages = np.repeat(rng.uniform(-3.0, 0.1, n // 32).astype(np.float32), 32)
    ages[32:64] = -0.0
    ages[64:96] = np.uint32(0xFFFFFFFF).view(np.float32)
    ages[97] = 0.25
    w = World(n, cap, chunks, k, monkeypatch, lifetimes=life, ages=ages, seed=3)
    for step in range(6):
        w.ref.sim.delta_time = np.float32(0.0 if step in (1, 2) else 1 / 60)
        w.frame(orc)
        d = w.check(f"frame {step}")
        assert not d[2] and not d[3], "all-ones and differing ages never defer"


@pytest.mark.parametrize("first,count", [(0, 4096), (40, 100), (5, 27), (33, 1), (4000, 96), (100, 0)])
def test_flush_kernel(first, count):
    """k_flush_group_ages over ranges that start and end inside groups: every deferred group the range touches gets its
    age in all 32 rows (none past the capacity), a writer's flush leaves the sentinel in every word and floor of the range,
    a reader's flush leaves deferred words known at its epoch; nothing outside the range changes."""
    cap = 4090
    rng = np.random.default_rng(first * 7 + count)
    columns = [[0, 1, 2, 4], [5, 6], [3], [7]]
    groups = cap // 32 + 1
    kinds = rng.integers(0, 3, groups)
    ages = rng.integers(0, 2**32, groups, dtype=np.uint64)
    words0 = np.where(kinds == 0, WORD_NONE, np.where(kinds == 1, (np.uint64(77) << np.uint64(32)) | ages,
                                                        np.uint64(1 << 62) | ages)).astype(np.uint64)
    words0 = np.append(words0, np.uint64((kinds == 2).sum()))  # the count of deferred words
    planes0 = [rng.integers(0, 2**32, cap * len(c), dtype=np.uint64).astype(np.uint32) for c in columns]
    floors0 = rng.integers(0, 2**32, groups, dtype=np.uint64).astype(np.uint32)
    g0, g1 = first // 32, (first + count + 31) // 32 if count else first // 32
    for clear in (True, False):
        planes, words, floors = [p.copy() for p in planes0], words0.copy(), floors0.copy()
        ps = plane_set(planes, columns)
        flush_lib().semu_flush_group_ages(C.byref(ps), AGE_WORD, words.ctypes.data, floors.ctypes.data, first, count, cap, int(clear), 123)
        want_age, want_words, want_floors = planes0[AGE_COL].copy(), words0.copy(), floors0.copy()
        for g in range(g0, g1):
            if kinds[g] == 2:
                want_words[-1] -= np.uint64(1)
                want_age[g * 32:min(cap, g * 32 + 32)] = np.uint32(int(ages[g]) & 0xFFFFFFFF)
            if clear:
                want_words[g], want_floors[g] = WORD_NONE, NONE
            elif kinds[g] == 2:
                want_words[g] = (np.uint64(123) << np.uint64(32)) | (ages[g] & np.uint64(0xFFFFFFFF))
        np.testing.assert_array_equal(planes[AGE_COL], want_age)
        np.testing.assert_array_equal(words, want_words)
        np.testing.assert_array_equal(floors, want_floors)
        for p in (0, 1, 3):
            np.testing.assert_array_equal(planes[p], planes0[p])
