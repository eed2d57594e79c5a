"""The tile shapes of tests/test_gpu_tile_shapes.py on the real kernel templates under the CPU thread emulation: K = 2 with 8
sub-tiles and K = 1 with 16 per tile for the authored effects of every record width, C5 with K forced to 1 and 2, and the
identity-claim edges at those shapes. Every buffer bit for bit against the oracle after every frame."""
import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import recipes
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.helpers import Instance
from tests.kernel_emu import EmuWorld
from tests.test_gpu_identity_claim import CLAIM_EDGE_SPAWNS, claim_edge_world
from tests.test_gpu_tile_shapes import EFFECTS, ROWS_PER_LANE, _asset, _edge_counts, _world, tile_k
from tests.test_identity_claim_emu_cpu import _claim, _claimed, _frame, claimed_driver  # noqa: F401
from tests.test_kernel_emu_cpu import _assert_same, _c5_world

pytestmark = pytest.mark.timeout(600)


@pytest.fixture(autouse=True)
def _default_shape(monkeypatch):
    for v in ("HNB_TILE_K", "HNB_ROWS_PER_LANE", "HNB_DEFINES"):
        monkeypatch.delenv(v, raising=False)


@pytest.mark.parametrize("name", list(EFFECTS))
def test_largest_tile_of_every_record_width(orc, name):
    """One batch of instances whose alive counts sit at the sub-tile and tile edges of the largest tile (8 sub-tiles at
    K = 2, 16 at K = 1): a burst of exactly that count, deaths, a burst into the shuffled dead stack."""
    k = tile_k(EFFECTS[name][1])
    chunks = ROWS_PER_LANE // k
    counts = _edge_counts(k, chunks)
    ref = _world(name, [n + 96 for n in counts])
    asset = _asset(name, max(counts) + 96)
    props = EFFECTS[name][3]
    blobs = None
    if props is not None:
        blobs = [asset.serialize_properties(props(i)) for i in range(len(counts))]
        for i in range(len(counts)):
            ref.metadata[i].properties_array_index = i
    eo = EffectOracle(asset, {i: props(i) for i in range(len(counts))} if props else None)
    emu = EmuWorld(ref, asset.generate(), chunks=chunks, update_ctas=2, property_blobs=blobs)
    assert emu.lib.emu_tile_k() == k and emu.tile == 32 * k * chunks
    schedule = [counts] + [[0] * len(counts)] * 6 + [[80] * len(counts), [0] * len(counts)]
    for f, spawns in enumerate(schedule):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        seeds = [int(s) for s in pcg_hash(np.arange(len(spawns), dtype=np.uint32) + np.uint32(100 * f + 7))]
        ref.set_spawns(spawns, seeds)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawns, seeds)
        _assert_same(ref, emu.pull(), f"{name} at {chunks} sub-tiles, frame {f}")
    assert all(ref.metadata[i].particle_counter == n + 80 for i, n in enumerate(counts))


@pytest.mark.parametrize("k", [1, 2])
def test_c5_with_k_forced(orc, monkeypatch, k):
    """C5's 32-byte records at K = 1 (16 sub-tiles) and K = 2 (8 sub-tiles) instead of its own K = 4."""
    monkeypatch.setenv("HNB_TILE_K", str(k))
    chunks = ROWS_PER_LANE // k
    rng = np.random.default_rng(k)
    ref = _c5_world(rng, [Instance(0, 5000, alive=4700, seed=42), Instance(5000, 700, alive=511, seed=43)])
    emu = EmuWorld(ref, recipes.c5_lowered(), chunks=chunks, update_ctas=2)
    assert emu.lib.emu_tile_k() == k
    accel_drag = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    for step in range(5):
        ref.oracle_frame(orc, orc.orc_body_update_c5(), accel_drag)
        emu.frame_step(orc, ref.sim, [0, 0], [42, 43])
        _assert_same(ref, emu.pull(), f"K {k}, step {step}")
    assert 0 < ref.metadata[0].alive_count < 4700


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("end", ["sub-1", "sub+1", "S-1", "S+1"])
def test_c5_claim_ending_at_tile_edges_with_k_forced(orc, claimed_driver, monkeypatch, k, end):
    """The claim-edge scenario at the largest tile of K = 1 and K = 2, with the claim words asserted after every frame:
    kept, shrunk to the first appended row by the burst, then dropped."""
    monkeypatch.setenv("HNB_TILE_K", str(k))
    chunks = ROWS_PER_LANE // k
    sub, S = 32 * k, 32 * k * chunks
    L = {"sub-1": sub - 1, "sub+1": sub + 1, "S-1": S - 1, "S+1": S + 1}[end]
    cap = L + 1100
    ref = claim_edge_world(L, cap)
    emu, claims = _claimed(ref, chunks, cap)
    assert emu.lib.emu_tile_k() == k
    for f, spawn in enumerate(CLAIM_EDGE_SPAWNS):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        _frame(orc, ref, emu, spawn)
        _assert_same(ref, emu.pull(), f"claim ending at row {L}, frame {f}")
        written = ref.metadata[0].indirect_write_index
        want = {0: (_claim(0, cap), _claim(0, cap)), 1: (0, _claim(0, L))}.get(f, (0, 0))
        assert (claims[written], claims[1 - written]) == want, f"claim ending at row {L}, frame {f}: claim words"
    assert ref.metadata[0].alive_count == 1000


@pytest.mark.parametrize("value,want", [("64", 32), ("33", 32), ("32", 32), ("8", 8)])
def test_rows_per_lane_is_clamped_to_32(monkeypatch, value, want):
    """Slot order gives each lane one 32-slot word of the alive bitmap: a tile may span at most 32 words, so a lane handles
    at most 32 rows of it, whatever HNB_ROWS_PER_LANE asks for."""
    monkeypatch.setenv("HNB_ROWS_PER_LANE", value)
    for fx in (recipes.c5_lowered(), recipes.c5_lowered(slot_order=True)):
        defines = [line for line in fx.generate_source().splitlines() if line.startswith("#define HNB_ROWS_PER_LANE ")]
        assert defines[0] == f"#define HNB_ROWS_PER_LANE {want}"
