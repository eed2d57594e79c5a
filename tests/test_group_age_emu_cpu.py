"""Common ages (DESIGN.md §3) on the real hnb_init / hnb_update kernels under the CPU thread emulation: beside each lifetime
floor the update keeps the age bits every row of the 32-row group holds, tagged with the frame's epoch, reads no age column
where the previous frame's update stored that word, and every result stays bit-identical to the oracle.

Every test runs at K = 1, 2, 4 and 8 rows in flight per lane (HNB_TILE_K), with 1, 2 and the most sub-tiles a tile holds.
Only here can a test poison an age column under a known word: on the device that takes a device view, which switches the
slab's floors and common ages off for good."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from bevy_hanabi_b200 import graph as G, recipes
from tests.effects import ROWS_PER_LANE
from tests.helpers import Instance
from tests.kernel_emu import CLAIMED_DRIVER, EmuWorld, assert_same, c5_frame, c5_world, claim

pytestmark = pytest.mark.timeout(600)

NONE = np.uint32(0xFFFFFFFF)
WORD_NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
RO_REAP = 1 | 2  # HNB_ATTR_UPDATE_READ_ONLY | HNB_ATTR_REAP_ONLY
SHAPES = [(k, n) for k in (1, 2, 4, 8) for n in sorted({1, 2, ROWS_PER_LANE // k})]
TILE_SHAPES = pytest.mark.parametrize("k,chunks", SHAPES, ids=[f"K{k}-{n}sub" for k, n in SHAPES])
AGE_COL = 2  # column [24, 28) of the C5 word map holds the age alone


@pytest.fixture(autouse=True)
def _default_shape(monkeypatch):
    for v in ("HNB_TILE_K", "HNB_ROWS_PER_LANE", "HNB_DEFINES"):
        monkeypatch.delenv(v, raising=False)


# The emulation driver with identity claims whose launches also pass the slab's floors and common ages.
_PARAMS = """static hnb::BatchParams make_params(const EmuBatch* b) {
    hnb::BatchParams P;
    memset((void*)&P, 0, sizeof(P));
"""
assert CLAIMED_DRIVER.count(_PARAMS) == 1
AGE_DRIVER = CLAIMED_DRIVER.replace(_PARAMS, """static float* g_life_floor = nullptr;
static unsigned long long* g_group_age = nullptr;
extern "C" void emu_set_group_words(float* floors, unsigned long long* ages) { g_life_floor = floors; g_group_age = ages; }
""" + _PARAMS + """    P.life_floor = g_life_floor;
    P.group_age = g_group_age;
""")


def c5_with_floors():
    """C5 with a read-only, reap-only lifetime: what the graph lowering makes of recipes.c5_asset."""
    fx = recipes.c5_lowered()
    return dataclasses.replace(fx, attrs=[dataclasses.replace(a, flags=RO_REAP if a.name == "lifetime" else 0) for a in fx.attrs])


def test_c5_word_map():
    fx = recipes.c5_asset(64).generate()
    assert fx.column_plan() == [(0, 16), (16, 8), (24, 4), (28, 4)]
    assert fx.column_words() == [[0, 1, 2, 4], [5, 6], [3], [7]]
    src = fx.generate_source()
    assert "\n#define HNB_LIFE_FLOOR 1\n" in src and "\n#define HNB_GROUP_AGE 1\n" in src
    assert c5_with_floors().column_words() == fx.column_words()


def _identity(fx):
    return all(words == list(range(o // 4, (o + w) // 4)) for words, (o, w) in zip(fx.column_words(), fx.column_plan()))


def test_only_effects_with_floors_get_word_maps():
    """The effects of tests/effects.py and the recipes: those that keep floors in a C5-like layout get the word map (and
    common ages); every other one keeps an identity map."""
    from tests import effects as E
    mapped = {"c5_asset": recipes.c5_asset(4096).generate(), "force_field": E.force_field(4096).generate(),
              "drifting_sparks": E.drifting_sparks(4096).generate(), "vec4x2_64": E.table_asset("vec4x2_64", 4096).generate(),
              "vec4x4_96": E.table_asset("vec4x4_96", 4096).generate()}
    identity = {"c5_lowered": recipes.c5_lowered(), "firework_trails": E.firework_trails(4096).generate(),
                "growing_dust": E.growing_dust(4096).generate(), "ribbon_asset": E.ribbon_asset(4096).generate(),
                "instancing": E.instancing(4096).generate(), "matrix_asset": E.matrix_asset(4096).generate(),
                "event_parent": E.event_assets()[0].generate(num_event_bindings=1),
                "event_child": E.event_assets()[1].generate(parent=E.event_assets()[0]),
                "emitter_parent": E.emitter_assets(4096)[0].generate(num_event_bindings=2)}
    for name, fx in mapped.items():
        src = fx.generate_source()
        assert not _identity(fx) and "\n#define HNB_GROUP_AGE 1\n" in src, name
        age, life = ({a.name: a.offset // 4 for a in fx.attrs}[n] for n in ("age", "lifetime"))
        assert [age] in fx.column_words() and [life] in fx.column_words(), name
    for name, fx in identity.items():
        assert _identity(fx) and "HNB_GROUP_AGE 1" not in fx.generate_source(), name


def test_update_that_writes_age_keeps_no_group_ages():
    """An update modifier that writes AGE: the lifetime is not reap-only, so neither floors nor common ages are kept, and the
    plan is the runs of written / read-only words."""
    w = G.ExprWriter()
    fx = (G.EffectAsset(64, w.module, name="rejuvenate")
          .init(G.SetAttributeModifier(G.Attribute.POSITION, w.lit(G.Vec3(0, 0, 0))))
          .init(G.SetAttributeModifier(G.Attribute.VELOCITY, w.lit(G.Vec3(0, 1, 0))))
          .init(G.SetAttributeModifier(G.Attribute.AGE, w.lit(0.)))
          .init(G.SetAttributeModifier(G.Attribute.LIFETIME, w.lit(2.)))
          .update(G.SetAttributeModifier(G.Attribute.AGE, w.attr(G.Attribute.AGE) * w.lit(0.5)))).generate()
    src = fx.generate_source()
    assert "HNB_LIFE_FLOOR 1" not in src and "HNB_GROUP_AGE 1" not in src
    assert _identity(fx)


def _world(n, cap, chunks, k, monkeypatch, lifetimes=None, ages=None, seed=1):
    monkeypatch.setenv("HNB_TILE_K", str(k))
    ref = c5_world(np.random.default_rng(seed), [Instance(0, cap, alive=n, seed=42)])
    ref.particles[:n, 7] = np.asarray(lifetimes if lifetimes is not None else np.full(n, 5.0), dtype=np.float32).view(np.uint32)
    if ages is not None:
        ref.particles[:n, 3] = np.asarray(ages, dtype=np.float32).view(np.uint32)
    fx = c5_with_floors()
    assert "#define HNB_GROUP_AGE 1" in fx.generate_source()
    emu = EmuWorld(ref, fx, chunks=chunks, update_ctas=2, driver=AGE_DRIVER)
    assert emu.lib.emu_tile_k() == k and emu.tile == 32 * k * chunks
    claims = np.array([claim(0, n)] * 2, dtype=np.uint64)  # as hnb_slab_fill_c5 leaves them
    emu.lib.emu_set_ident_claim.argtypes = [C.c_void_p]
    emu.lib.emu_set_ident_claim.restype = None
    emu.lib.emu_set_ident_claim(claims.ctypes.data)
    emu.claims = claims  # the kernels update it in place: it must live as long as the world
    floors = np.full(cap // 32 + 1, NONE, dtype=np.uint32)
    ages_w = np.full(cap // 32 + 1, WORD_NONE, dtype=np.uint64)
    emu.lib.emu_set_group_words.argtypes = [C.c_void_p, C.c_void_p]
    emu.lib.emu_set_group_words.restype = None
    emu.lib.emu_set_group_words(floors.ctypes.data, ages_w.ctypes.data)
    return ref, emu, floors, ages_w


def _age(words):
    """The age bits of common-age words."""
    return (np.asarray(words) & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def _epoch(words):
    return (np.asarray(words) >> np.uint64(32)).astype(np.uint32)


def _floor_groups(emu, n):
    """Groups of the tiles wholly below a claim of n rows: the only ones whose words the update reads or stores."""
    return (n // emu.tile) * emu.tile // 32


@TILE_SHAPES
def test_ages_known_then_never_loaded(orc, monkeypatch, k, chunks):
    """Frame 0 stores every floor group's common age (the fill's 0 plus dt). Then the age column is poisoned with NaN payloads
    under the known words: the update never reads it, and the ages it stores are the oracle's."""
    n, cap = 2900, 3200
    ref, emu, _, ages = _world(n, cap, chunks, k, monkeypatch)
    c5_frame(orc, ref, emu)
    assert_same(ref, emu.pull(), "frame 0")
    full = _floor_groups(emu, n)
    assert full > 0
    np.testing.assert_array_equal(_age(ages[:full]), np.full(full, np.float32(ref.sim.delta_time)).view(np.uint32))
    assert (_epoch(ages[:full]) == emu.epoch).all() and (ages[full:] == WORD_NONE).all()
    col = emu.planes[AGE_COL]
    col[:full * 32] = np.uint32(0x7FC0DEAD)
    for step in range(1, 4):
        c5_frame(orc, ref, emu)
        assert_same(ref, emu.pull(), f"frame {step}")
    np.testing.assert_array_equal(_age(ages[:full]), ref.particles[:full * 32:32, 3])


@TILE_SHAPES
def test_differing_ages_and_all_ones(orc, monkeypatch, k, chunks):
    """A group with one differing age stores nothing and stays unknown; a group whose ages are all ones (the sentinel's
    bits) never becomes known; every other floor group is stored at each frame's epoch."""
    n, cap = 2048, 2048
    ages = np.zeros(n, dtype=np.float32)
    ages[37] = 0.25                                        # group 1: one row differs
    ages[64:96] = np.uint32(0xFFFFFFFF).view(np.float32)  # group 2: all ones
    ref, emu, _, words = _world(n, cap, chunks, k, monkeypatch, ages=ages, seed=2)
    full = _floor_groups(emu, n)
    for step in range(3):
        c5_frame(orc, ref, emu)
        assert_same(ref, emu.pull(), f"frame {step}")
        assert words[1] == WORD_NONE and words[2] == WORD_NONE
        if ref.metadata[0].alive_count == n or step == 0:
            assert _epoch(words[0]) == emu.epoch and (_epoch(words[3:full]) == emu.epoch).all()


@pytest.mark.parametrize("k", [1, 2, 4, 8], ids=lambda k: f"K{k}")
def test_tile_size_changes_between_frames(orc, monkeypatch, k):
    """The tile size of a launch follows the slab and the batch, so it may change from frame to frame, and with it which
    groups lie in floor tiles. A group updated outside a floor tile keeps the word of an older epoch: it is never read as
    known again, and the age column is loaded (using it would store the age of an earlier frame plus dt, which the oracle
    comparison shows)."""
    n, cap = 1000, 4096
    ref, emu, _, words = _world(n, cap, 1, k, monkeypatch)
    most = ROWS_PER_LANE // k
    chunk_seq = [c for c in (1, most, 2, most, 1, 3, most, 2, 1, most) if c <= most]
    for f, chunks in enumerate(chunk_seq):
        emu.tile_word = 32 * k * chunks
        emu.b.tile_rows = emu.tile_word
        emu.tile = emu.tile_word
        c5_frame(orc, ref, emu)
        assert_same(ref, emu.pull(), f"frame {f}, {chunks} sub-tiles")
        full = (n // emu.tile) * emu.tile // 32
        assert (_epoch(words[:full]) == emu.epoch).all()
        assert not (_epoch(words[full:]) == emu.epoch).any()
@TILE_SHAPES
def test_special_values(orc, monkeypatch, k, chunks):
    """Common negative ages, -0.0, NaN and infinite lifetimes, and frames with dt = 0, against the oracle."""
    n, cap = 2048, 2048
    rng = np.random.default_rng(9)
    life = rng.uniform(0.2, 2.0, n).astype(np.float32)
    life[rng.choice(n, 12, replace=False)] = np.nan
    life[rng.choice(n, 12, replace=False)] = np.inf
    life[rng.choice(n, 12, replace=False)] = -np.inf
    ages = np.repeat(rng.uniform(-3.0, 0.1, n // 32).astype(np.float32), 32)
    ages[32:64] = -0.0
    ref, emu, _, words = _world(n, cap, chunks, k, monkeypatch, lifetimes=life, ages=ages, seed=3)
    for step in range(6):
        ref.sim.delta_time = np.float32(0.0 if step in (1, 2) else 1 / 60)
        c5_frame(orc, ref, emu)
        assert_same(ref, emu.pull(), f"frame {step}")
        if ref.metadata[0].alive_count == n:
            full = _floor_groups(emu, n)
            np.testing.assert_array_equal(_age(words[:full]), ref.particles[:full * 32:32, 3])


@pytest.mark.parametrize("k", [1, 2, 4, 8], ids=lambda k: f"K{k}")
def test_init_clears_the_group_of_each_slot_it_writes(orc, monkeypatch, k):
    """Spawns into slots whose groups hold a (here wrong) common age set those words to the sentinel."""
    n, cap = 1000, 2048
    ref, emu, _, words = _world(n, cap, 1, k, monkeypatch)
    groups = np.unique(np.arange(n, n + 300) // 32)  # init appends slots n .. n+299 (the dead stack is the identity)
    words[groups] = np.uint64(0) | np.uint64(np.float32(-7.0).view(np.uint32))  # the epoch the first frame reads as known
    c5_frame(orc, ref, emu, spawn=300)
    assert_same(ref, emu.pull(), "spawn frame")
    assert (words[groups] == WORD_NONE).all()
