"""Lifetime floors (DESIGN.md §3) of the authored C5 (recipes.c5_asset: its own column plan [0,16) [16,24) [24,28) [28,32) and
HNB_LIFE_FLOOR 1, the module bench.py times) against the C oracle at every tile shape: K = 1, 2, 4 and 8 rows in flight per
lane, with 1, 2 and the most sub-tiles a tile holds, at 16 and at 32 rows per lane. The code under test runs only there: the
floor load of lanes k < K, the slab group g_first + k of row group k of sub-tile j, its broadcast from lane k and its store.
A floor of the wrong group stays silent wherever lifetimes are uniform and kills particles late where they are not.

Every world starts from hnb_slab_fill_c5 on the device and orc_fill_c5 in the oracle, over the same counter-based state:
the fill is the writer that gives an instance its identity claim. Records, both alive lists, the dead stack and every
counter are compared row by row after every frame, and each test reads back the tile size it claims to cover. Whether
floors really engage (rows proven alive without a lifetime load) is shown by tests/test_lifetime_floor_emu_cpu.py at the
same shapes: on the device only a device view can poison a lifetime column, and a device view switches floors off.

Also: the authored effects of tests/effects.py that keep floors at K = 2 and K = 1, against the numpy oracle."""
from dataclasses import dataclass

import numpy as np
import pytest

from tests.effects import EFFECTS, table_asset, table_props, tile_k
from tests.helpers import Instance, Lockstep, filled_c5, is_identity, seeds, table_world
from tests.repack_ref import ref_repack

pytestmark = pytest.mark.gpu


@dataclass(frozen=True)
class Shape:
    k: int            # rows in flight per lane (HNB_TILE_K)
    chunks: int       # sub-tiles of 32 K rows per tile (HNB_TILE_CHUNKS)
    rows_per_lane: int

    @property
    def tile(self):
        return 32 * self.k * self.chunks


SHAPES = [Shape(k, n, rpl) for rpl in (16, 32) for k in (1, 2, 4, 8) for n in sorted({1, 2, rpl // k})]


def _force(mp, k, chunks, rows_per_lane=None):
    mp.setenv("HNB_TILE_K", str(k))
    mp.setenv("HNB_TILE_CHUNKS", str(chunks))
    if rows_per_lane is None:
        mp.delenv("HNB_ROWS_PER_LANE", raising=False)
    else:
        mp.setenv("HNB_ROWS_PER_LANE", str(rows_per_lane))
    if k == 8:
        mp.setenv("HNB_DEFINES", "HNB_MIN_BLOCKS=2")  # 8 rows in flight per lane do not fit the default register budget
    else:
        mp.delenv("HNB_DEFINES", raising=False)


@pytest.fixture(scope="module", params=SHAPES, ids=[f"K{s.k}-{s.chunks}sub-{s.rows_per_lane}rpl" for s in SHAPES])
def shaped(request, native):
    """(context, the authored C5 compiled in it) at one forced shape: one context and one module serve every scenario."""
    from bevy_hanabi_b200 import recipes
    s = request.param
    with pytest.MonkeyPatch.context() as mp:
        _force(mp, s.k, s.chunks, s.rows_per_lane)
        fx = recipes.c5_asset(1 << 20).generate()
        src = fx.generate_source()
        assert f"\n#define HNB_TILE_K {s.k}\n" in src and f"\n#define HNB_ROWS_PER_LANE {s.rows_per_lane}\n" in src
        assert "\n#define HNB_LIFE_FLOOR 1\n" in src
        assert fx.column_plan() == [(0, 16), (16, 8), (24, 4), (28, 4)]
        c = native.Context(0)
        try:
            yield c, c.effect_compile(fx), s
        finally:
            c.close()


@pytest.fixture
def fctx(shaped):
    """The shaped context for one test; afterwards batch 0's last update must have run at the shape's tile size."""
    c, effect, s = shaped
    c.authored, c.shape = effect, s
    yield c
    assert c.read_tile_size(0) == s.tile, "the update ran at another tile size than the one under test"


def _set_dt(ref, dt):
    ref.sim.delta_time = ref.sim.virtual_delta_time = ref.sim.real_delta_time = np.float32(dt)


def _lock(ctx, orc, insts, fills):
    return filled_c5(ctx, orc, insts, fills, effect=ctx.authored)


def test_lifetimes_1_to_3(fctx, orc):
    """C5 variant B for 150 frames: floors are stored on frame 0, nobody dies for about 60 frames while they prove rows
    alive, then deaths fall inside groups and end the claim."""
    n = 4096 + 77
    lock = _lock(fctx, orc, [Instance(0, n, alive=n, seed=42)], [(0, n, 1234, 1.0, 3.0)])
    lock.run(55, what="before the first death")
    assert lock.ref.metadata[0].alive_count == n
    lock.run(95, start=55, what="deaths")
    assert 0 < lock.ref.metadata[0].alive_count < n


@pytest.mark.parametrize("end", ["S-1", "S+1", "G-1", "G+1"])
def test_claim_ending_next_to_an_edge(fctx, orc, end):
    """The claim (fill and alive count) ends one row before or after a tile edge (S) or a 32-row group edge inside the
    third tile (G = 2S + 32); deaths from frame 30 on, two bursts into the freed slots."""
    S = fctx.shape.tile
    L = {"S-1": S - 1, "S+1": S + 1, "G-1": 2 * S + 31, "G+1": 2 * S + 33}[end]
    cap = L + S + 300
    lock = _lock(fctx, orc, [Instance(0, cap, alive=L, seed=7)], [(0, L, 99, 0.5, 1.5)])
    schedule = [[0]] * 10 + [[S // 2 + 7]] + [[0]] * 59 + [[200]] + [[0]] * 29
    lock.run(schedule, what=f"claim ending at row {L}")
    md = lock.ref.metadata[0]
    assert md.particle_counter == S // 2 + 7 + 200 and md.alive_count == 200  # the fill and the first burst died


def test_instance_off_a_group(fctx, orc):
    """The claimed instance starts at slab row 40, inside a 32-row group: it keeps no floors and must still be exact."""
    S = fctx.shape.tile
    cap1 = 3 * S + 100
    insts = [Instance(0, 40, alive=40, seed=5), Instance(40, cap1, alive=cap1 - 50, seed=6)]
    lock = _lock(fctx, orc, insts, [(0, 40, 3, 0.2, 0.9), (40, cap1 - 50, 4, 0.3, 1.0)])
    schedule = [[0, 0]] * 30 + [[10, 40]] + [[0, 0]] * 39
    lock.run(schedule, what="off a group")
    assert 0 < lock.ref.metadata[1].alive_count < cap1 - 50


def test_claim_held_by_the_second_instance(fctx, orc):
    """Two instances in one batch, the second filled last so that it holds the claim: its floor groups start at slab row
    S + 96, a group edge off the tile grid, and its tiles after the first instance's."""
    S = fctx.shape.tile
    c0, c1 = S + 96, 4 * S + 64
    insts = [Instance(0, c0, alive=c0, seed=8), Instance(c0, c1, alive=c1 - 30, seed=9)]
    lock = _lock(fctx, orc, insts, [(0, c0, 10, 0.2, 0.6), (c0, c1 - 30, 11, 1.0, 2.0)])
    schedule = [[0, 0]] * 40 + [[50, 0]] + [[0, 0]] * 39 + [[0, 100]] + [[0, 0]] * 49
    lock.run(schedule, what="claim held by instance 1")
    assert 0 < lock.ref.metadata[1].alive_count < c1 - 30


def test_special_values_and_zero_dt(fctx, orc):
    """NaN, infinite and negative lifetimes (in the upper half, so that the claim keeps the lower half), negative and -0
    ages, whole groups of +inf lifetimes, and frames with dt = 0. The records are uploaded after the fill, which clears the
    floors and keeps the claim."""
    n = 2048 + 45
    lock = _lock(fctx, orc, [Instance(0, n, alive=n, seed=12)], [(0, n, 77, 0.1, 2.0)])
    ref = lock.ref
    rng = np.random.default_rng(fctx.shape.tile + fctx.shape.k)
    life, age = ref.particles[:, 7].view(np.float32), ref.particles[:, 3].view(np.float32)
    half = n // 2
    up = lambda m: half + rng.choice(n - half, m, replace=False)  # noqa: E731
    life[up(20)] = np.nan
    life[up(20)] = np.inf
    life[up(20)] = -np.inf
    life[up(40)] = rng.uniform(-1.0, 0.0, 40)
    life[half + 32 - half % 32:half + 64 - half % 32] = np.nan  # a whole group of NaNs: its floor proves nothing
    life[64:96] = np.inf                                         # a whole group of +inf: proven forever
    life[rng.choice(half, 16, replace=False)] = np.inf
    age[rng.choice(n, 256, replace=False)] = rng.uniform(-2.0, 0.0, 256)
    age[rng.choice(n, 16, replace=False)] = -0.0
    fctx.slab_upload_aos(lock.gpu.slab, 0, ref.particles)
    for f in range(24):
        _set_dt(ref, 0.0 if f in (2, 3, 11) else 1.0 / 60.0)
        lock.run([[0]], start=f, what="special values")
    assert 0 < ref.metadata[0].alive_count < n


# ---- authored effects with floors at K = 2 and K = 1 -------------------------------------------------------------------
@pytest.mark.parametrize("name,chunks", [("vec4x2_64", 1), ("vec4x2_64", 8), ("vec4x4_96", 1), ("vec4x4_96", 16)],
                         ids=["vec4x2_64-1sub", "vec4x2_64-8sub", "vec4x4_96-1sub", "vec4x4_96-16sub"])
def test_wide_records_with_floors(native, orc, monkeypatch, name, chunks):
    """64-byte (K = 2) and 96-byte (K = 1) records, whose lifetimes have 4-byte columns of their own, against the numpy
    oracle: a burst, a repack that gives the instance its claim, frames in which floors prove rows alive, deaths inside
    groups and spawns into the freed slots."""
    k = tile_k(EFFECTS[name][1])
    cap = 3000
    asset = table_asset(name, cap)
    monkeypatch.setenv("HNB_TILE_CHUNKS", str(chunks))
    for v in ("HNB_TILE_K", "HNB_ROWS_PER_LANE", "HNB_DEFINES"):
        monkeypatch.delenv(v, raising=False)
    src = asset.generate().generate_source()
    assert "\n#define HNB_LIFE_FLOOR 1\n" in src and f"\n#define HNB_TILE_K {k}\n" in src
    ref = table_world(name, [cap])
    _set_dt(ref, 0.02)  # lifetimes U(0.25, 0.6): 12 to 30 frames
    c = native.Context(0)
    try:
        lock = Lockstep(c, orc, ref, asset, props=table_props(name, 1), seeds=seeds)
        lock.run([[2600]], what=f"{name} burst")
        assert not is_identity(ref, 0)
        c.slab_repack(lock.gpu.slab, lock.gpu.effect, 0, 0, cap)
        ref_repack(ref, 0)
        lock.compare("after the repack")
        schedule = [[0]] * 14 + [[150]] + [[0]] * 5 + [[300]] + [[0]] * 9
        lock.run(schedule, start=1, what=name)
        assert ref.metadata[0].particle_counter == 2600 + 150 + 300 and ref.metadata[0].alive_count < 2600 + 450
        assert c.read_tile_size(0) == 32 * k * chunks
    finally:
        c.close()
