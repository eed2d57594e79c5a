"""Lifetime floors (DESIGN.md §3) on the real hnb_init / hnb_update kernels under the CPU thread emulation: the update stores a
floor per 32 rows of an identity-claimed tile, proves rows alive from it without loading their lifetimes, and every result
stays bit-identical to the oracle, including NaN, infinite and negative lifetimes, negative ages and dt = 0.

Every test runs at K = 1, 2, 4 and 8 rows in flight per lane (HNB_TILE_K), with 1, 2 and the most sub-tiles a tile holds:
the floor load of lanes k < K, the slab group g_first + k of row group k of sub-tile j, its broadcast and its store. Only
here can a test show that floors really engage: the poisoned-lifetime test overwrites lifetimes the floor proves alive,
which on the device takes a device view, and a device view switches the slab's floors off for good
(tests/test_gpu_floor_shapes.py covers the same shapes on the device against the oracle)."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from bevy_hanabi_b200 import recipes
from tests.effects import ROWS_PER_LANE
from tests.helpers import Instance
from tests.kernel_emu import CLAIMED_DRIVER, EmuWorld, assert_same, c5_frame, c5_world, claim

pytestmark = pytest.mark.timeout(600)

NONE = np.uint32(0xFFFFFFFF)
RO_REAP = 1 | 2  # HNB_ATTR_UPDATE_READ_ONLY | HNB_ATTR_REAP_ONLY
# (K, sub-tiles per tile): 1, 2 and the most a tile holds at the default 16 rows per lane. K = 4 (C5's own) keeps the ids it
# had before K was forced.
SHAPES = [(k, n) for k in (1, 2, 4, 8) for n in sorted({1, 2, ROWS_PER_LANE // k})]
TILE_SHAPES = pytest.mark.parametrize("k,chunks", SHAPES, ids=[f"{n}sub" if k == 4 else f"K{k}-{n}sub" for k, n in SHAPES])


@pytest.fixture(autouse=True)
def _default_shape(monkeypatch):
    for v in ("HNB_TILE_K", "HNB_ROWS_PER_LANE", "HNB_DEFINES"):
        monkeypatch.delenv(v, raising=False)

# The emulation driver with identity claims, whose launches also pass the slab's lifetime floors (BatchParams::life_floor;
# NULL until emu_set_life_floor names an array).
_PARAMS = """static hnb::BatchParams make_params(const EmuBatch* b) {
    hnb::BatchParams P;
    memset((void*)&P, 0, sizeof(P));
"""
assert CLAIMED_DRIVER.count(_PARAMS) == 1
FLOOR_DRIVER = CLAIMED_DRIVER.replace(_PARAMS, """static float* g_life_floor = nullptr;
extern "C" void emu_set_life_floor(float* floors) { g_life_floor = floors; }
""" + _PARAMS + """    P.life_floor = g_life_floor;
""")


def c5_with_floors():
    """C5 with a read-only, reap-only lifetime: what the graph lowering makes of recipes.c5_asset."""
    fx = recipes.c5_lowered()
    return dataclasses.replace(fx, attrs=[dataclasses.replace(a, flags=RO_REAP if a.name == "lifetime" else 0) for a in fx.attrs])


def _world(n, cap, chunks, k, monkeypatch, lifetimes=None, ages=None, seed=1):
    monkeypatch.setenv("HNB_TILE_K", str(k))
    ref = c5_world(np.random.default_rng(seed), [Instance(0, cap, alive=n, seed=42)])
    if lifetimes is not None:
        ref.particles[:n, 7] = np.asarray(lifetimes, dtype=np.float32).view(np.uint32)
    if ages is not None:
        ref.particles[:n, 3] = np.asarray(ages, dtype=np.float32).view(np.uint32)
    fx = c5_with_floors()
    src = fx.generate_source()
    assert "#define HNB_LIFE_FLOOR 1" in src and f"\n#define HNB_TILE_K {k}\n" in src
    emu = EmuWorld(ref, fx, chunks=chunks, update_ctas=2, driver=FLOOR_DRIVER)
    assert emu.lib.emu_tile_k() == k and emu.tile == 32 * k * chunks
    claims = np.array([claim(0, n)] * 2, dtype=np.uint64)  # as hnb_slab_fill_c5 leaves them
    emu.lib.emu_set_ident_claim.argtypes = [C.c_void_p]
    emu.lib.emu_set_ident_claim.restype = None
    emu.lib.emu_set_ident_claim(claims.ctypes.data)
    floors = np.full(cap // 32 + 1, NONE, dtype=np.uint32)
    emu.lib.emu_set_life_floor.argtypes = [C.c_void_p]
    emu.lib.emu_set_life_floor.restype = None
    emu.lib.emu_set_life_floor(floors.ctypes.data)
    return ref, emu, claims, floors


def _group_minima(lifetimes, groups):
    """NaN-propagating minimum of each full 32-row group."""
    g = np.asarray(lifetimes[:groups * 32], dtype=np.float32).reshape(groups, 32)
    return np.where(np.isnan(g).any(axis=1), np.float32(np.nan), g.min(axis=1))


def test_lowered_c5_gets_the_flag_and_hand_lowered_does_not():
    lt = {a.name: a.flags for a in recipes.c5_asset(64).generate().attrs}
    assert lt["lifetime"] == RO_REAP and lt["age"] == 0
    assert all(a.flags == 0 for a in recipes.c5_lowered().attrs)
    assert "HNB_LIFE_FLOOR 1" not in recipes.c5_lowered().generate_source()
    # on a default-cut slab the lifetime shares a column with velocity: no floors
    assert "HNB_LIFE_FLOOR 1" not in c5_with_floors().generate_source_for_plan([(0, 16), (16, 16)])


@TILE_SHAPES
def test_floors_are_stored_then_prove_rows_alive_without_loading(orc, monkeypatch, k, chunks):
    """Frame 0 stores each full group's minimum; from frame 1 on, rows the floor proves alive never read their lifetime
    (poisoned in the emulated slab, results still those of the oracle); deaths in the middle of groups drop the claim."""
    n, cap = 2900, 3200
    ref, emu, claims, floors = _world(n, cap, chunks, k, monkeypatch, lifetimes=np.random.default_rng(5).uniform(0.12, 0.6, n))
    c5_frame(orc, ref, emu)
    assert_same(ref, emu.pull(), "frame 0")
    tile = emu.tile
    full = (n // tile) * tile // 32  # groups of tiles wholly below the claim
    life = ref.particles[:n, 7].view(np.float32)
    np.testing.assert_array_equal(floors[:full].view(np.float32), _group_minima(life, full))
    assert (floors[full:] == NONE).all()
    # Poison the lifetimes of the rows the floor proves alive this frame: they must not be loaded.
    age, dt = ref.particles[:n, 3].view(np.float32), np.float32(ref.sim.delta_time)
    rows = np.arange(full * 32)
    f = floors[rows // 32].view(np.float32)
    proven = rows[(age[rows] < f) & (age[rows] + dt < f)]
    assert len(proven) > 0
    life_col = emu.planes[3].view(np.float32)  # column [28, 32) of the C5 plan
    life_col[proven] = np.float32(-1.0)
    c5_frame(orc, ref, emu)
    got = emu.pull()
    assert (got["particles"][proven, 7].view(np.float32) == -1.0).all()
    got["particles"][proven, 7] = ref.particles[proven, 7]
    assert_same(ref, got, "frame 1")
    life_col[proven] = life[proven]
    for step in range(2, 40):
        c5_frame(orc, ref, emu)
        assert_same(ref, emu.pull(), f"frame {step}")
        if ref.metadata[0].alive_count < n:
            break
    assert ref.metadata[0].alive_count < n, "deaths were expected"
    assert claims[ref.metadata[0].indirect_write_index] == 0


@TILE_SHAPES
def test_special_values(orc, monkeypatch, k, chunks):
    """NaN, infinite and negative lifetimes, negative ages, and frames with dt = 0, against the oracle."""
    n, cap = 2048, 2048
    rng = np.random.default_rng(9)
    life = rng.uniform(0.2, 2.0, n).astype(np.float32)
    life[rng.choice(n, 12, replace=False)] = np.nan
    life[rng.choice(n, 12, replace=False)] = np.inf
    life[rng.choice(n, 12, replace=False)] = -np.inf
    life[rng.choice(n, 40, replace=False)] = rng.uniform(-1.0, 0.0, 40)
    life[64:96] = np.nan  # a whole group of NaNs: its floor is NaN and proves nothing
    ages = rng.uniform(-3.0, 0.1, n).astype(np.float32)
    ages[rng.choice(n, 8, replace=False)] = -0.0
    ref, emu, _, floors = _world(n, cap, chunks, k, monkeypatch, lifetimes=life, ages=ages, seed=3)
    for step in range(6):
        ref.sim.delta_time = np.float32(0.0 if step in (1, 2) else 1 / 60)
        c5_frame(orc, ref, emu)
        assert_same(ref, emu.pull(), f"frame {step}")
        if step == 0:
            assert floors[2] != NONE and np.isnan(floors[2:3].view(np.float32)).all()


def test_init_clears_the_group_of_each_slot_it_writes(orc, monkeypatch):
    """Spawns into slots whose groups hold a floor (here a wrong one, far too high) set those groups to the sentinel."""
    _init_clears(orc, monkeypatch, 4)


@pytest.mark.parametrize("k", [1, 2, 8], ids=lambda k: f"K{k}")
def test_init_clears_the_group_of_each_slot_it_writes_at_other_k(orc, monkeypatch, k):
    _init_clears(orc, monkeypatch, k)


def _init_clears(orc, monkeypatch, k):
    n, cap = 1000, 2048
    ref, emu, _, floors = _world(n, cap, 1, k, monkeypatch)
    groups = np.unique(np.arange(n, n + 300) // 32)  # init appends slots n .. n+299 (the dead stack is the identity)
    floors[groups] = np.float32(1e30).view(np.uint32)
    c5_frame(orc, ref, emu, spawn=300)
    assert_same(ref, emu.pull(), "spawn frame")
    assert (floors[groups] == NONE).all()
