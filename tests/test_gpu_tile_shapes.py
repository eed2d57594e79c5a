"""The update pass at every tile shape on the device. A lane keeps K rows in flight per sub-tile of 32 x K rows, and K comes
from the record width: 4 up to 36 bytes (C5), 2 from 40 to 76 bytes, 1 from 80 bytes. A tile holds 1 up to
HNB_ROWS_PER_LANE / K sub-tiles: 4, 8 or 16 at the default 16 rows per lane. Code that only runs at K < 4 or beyond 4
sub-tiles: stash, ballot and bitmap-word indices j*K + k up to 15, the prefetch of the next sub-tile over 8 or 16 of them,
slot order's word ownership, per-warp Properties staging at K = 1, and the ordered-events row index.

Every buffer is compared bit for bit with the oracle after every frame, with IEEE-exact effects only (zero tolerance). The
results are the same at every tile shape by design, so each forced case reads the tile size back to prove which one ran."""
import numpy as np
import pytest

from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import recipes
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.helpers import GpuWorld, Instance, RefWorld, assert_world_equal
from tests.test_gpu_effects import _assert_relaxed_equal, _firework_trails
from tests import test_gpu_identity_claim as claims, test_gpu_ordered_events as ordered_events
from tests.test_gpu_identity_claim import CLAIM_EDGE_SPAWNS, _frames, claim_edge_world
from tests.test_gpu_slot_order import _run_c5
from tests.test_gpu_update_c5 import _fill
from tests.test_host_exec_cpu import _MATRIX_PROPS, _matrix_asset

pytestmark = pytest.mark.gpu
A = G.Attribute
ROWS_PER_LANE = 16  # HNB_ROWS_PER_LANE's default


def tile_k(stride):
    """choose_tile_k restated: rows a lane keeps in flight for records of `stride` bytes (index + record ~ 40 words)."""
    k = 40 // (stride // 4 + 1)
    return 4 if k >= 4 else 2 if k >= 2 else 1


def sub_tile_counts(k):
    """1, 2, 3, half the maximum + 1 and the maximum: {1, 2, 3, 5, 8} at K = 2, {1, 2, 3, 9, 16} at K = 1."""
    m = ROWS_PER_LANE // k
    return [1, 2, 3, m // 2 + 1, m]


@pytest.fixture
def shaped_ctx(request, native, monkeypatch):
    """A fresh context on cuda:0 with `chunks` sub-tiles per update tile forced by HNB_TILE_CHUNKS (request.param:
    `chunks` or `(chunks, K)`, K forced with HNB_TILE_K). The test sets `ctx.stride` (record bytes) and `ctx.batches`;
    afterwards every batch's last update must have used 32 x K x min(chunks, 16 / K) rows per tile."""
    chunks, forced_k = request.param if isinstance(request.param, tuple) else (request.param, None)
    monkeypatch.setenv("HNB_TILE_CHUNKS", str(chunks))
    monkeypatch.delenv("HNB_ROWS_PER_LANE", raising=False)
    if forced_k is None:
        monkeypatch.delenv("HNB_TILE_K", raising=False)
    else:
        monkeypatch.setenv("HNB_TILE_K", str(forced_k))
        if forced_k == 8:
            monkeypatch.setenv("HNB_DEFINES", "HNB_MIN_BLOCKS=2")  # 8 rows in flight per lane do not fit the default register budget
    c = native.Context(0)
    c.tile_chunks, c.forced_k, c.stride, c.batches = chunks, forced_k, None, [0]
    try:
        yield c
        k = forced_k or tile_k(c.stride)
        want = 32 * k * min(chunks, ROWS_PER_LANE // k)
        for b in c.batches:
            assert c.read_tile_size(b) == want, f"batch {b} ran at another tile size than the one under test"
    finally:
        c.close()


# ---- effects ----------------------------------------------------------------------------------------------------------
def _vec4s(capacity, n):
    """A 32-byte spark plus `n` vec4 attributes, each updated from itself, its neighbour and a per-instance property:
    64 bytes with 2 of them, 96 bytes with 4 (adds and multiplies only: IEEE-exact)."""
    w = G.ExprWriter()
    gain = w.prop(w.add_property("gain", 1.0))
    slots = [A.F32X4_0, A.F32X4_1, A.F32X4_2, A.F32X4_3][:n]
    asset = (G.EffectAsset(capacity, w.module, name=f"vec4x{n}")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.25).uniform(w.lit(0.6)))))
    for s in slots:
        asset = asset.init(G.SetAttributeModifier(s, w.rand(G.VEC4)))
    for i, s in enumerate(slots):
        asset = asset.update(G.SetAttributeModifier(s, w.attr(s) * w.lit(0.75) + w.attr(slots[i - 1]) * gain))
    return asset.update(G.AccelModifier(w.lit(G.Vec3(0., -3., 0.)) * gain))


# name -> (builder, record bytes, dt: lifetimes of 2-6 frames, properties of instance i or None)
EFFECTS = {
    "trails48": (_firework_trails, 48, 0.25, None),
    "vec4x2_64": (lambda cap: _vec4s(cap, 2), 64, 0.1, lambda i: {"gain": 0.5 + 0.125 * i}),
    "vec4x4_96": (lambda cap: _vec4s(cap, 4), 96, 0.1, lambda i: {"gain": 1.5 - 0.125 * i}),
    "matrix144": (_matrix_asset, 144, 0.15, lambda i: _MATRIX_PROPS if i % 2 == 0 else {}),
}


def _asset(name, capacity):
    build, size, _, _ = EFFECTS[name]
    asset = build(capacity)
    assert asset.particle_layout()[1] == size, f"{name}: record size"
    return asset


def _shapes(names):
    """(chunks, effect) for every effect of `names` at every sub-tile count of its K."""
    return [pytest.param(n, name, id=f"{name}-{n}sub") for name in names for n in sub_tile_counts(tile_k(EFFECTS[name][1]))]


ALL = list(EFFECTS)
SECTOR = ["trails48", "vec4x2_64", "vec4x4_96"]  # 32 + 16 B, 2 x 32 B and 3 x 32 B columns


def _world(name, caps, batches=None, align=1, dead_perm_seed=None):
    """A slab of instances of effect `name` with the given capacities, none alive, every dead stack shuffled."""
    _, size, dt, props = EFFECTS[name]
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=17 + 31 * i))
        off += (c + align - 1) // align * align
    ref = RefWorld(max(off, 1), size // 4, insts, batches=batches, dt=dt)
    rng = np.random.default_rng(dead_perm_seed if dead_perm_seed is not None else sum(caps))
    for inst in insts:
        rows = slice(inst.slab_offset, inst.slab_offset + inst.capacity)
        ref.indirect[rows, 2] = rng.permutation(ref.indirect[rows, 2])
    for i in range(len(insts)):  # per-instance emitter translations (Global simulation space adds them at init)
        tr = list(ref.spawners[i].transform)
        tr[3], tr[7], tr[11] = 0.5 * i, -0.25 * i, 1.0 + i
        for k in range(12):
            ref.spawners[i].transform[k] = tr[k]
    return ref


def _run(ctx, orc, name, ref, schedule, *, sector=False, slot=False, relaxed=False):
    """`schedule`: per frame, the spawn count of every instance. Returns the last pulled state."""
    asset = _asset(name, max(i.capacity for i in ref.instances))
    props = EFFECTS[name][3]
    blobs = None
    if props is not None:
        blobs = [asset.serialize_properties(props(i)) for i in range(len(ref.instances))]
        for i in range(len(ref.instances)):
            ref.metadata[i].properties_array_index = i
    ctx.stride, ctx.batches = asset.particle_layout()[1], list(range(len(ref.batches)))
    ref.slot_order = slot
    eo = EffectOracle(asset, {i: props(i) for i in range(len(ref.instances))} if props else None)
    gpu = GpuWorld(ctx, ref, asset.generate(sector_planes=sector, slot_order=slot, relaxed_order=relaxed), property_blobs=blobs,
                   sector_planes=sector)
    for f, spawns in enumerate(schedule):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns(spawns, [int(s) for s in pcg_hash(np.arange(len(spawns), dtype=np.uint32) + np.uint32(100 * f + 7))])
        eo.frame(ref, orc)
        gpu.frame()
        got = gpu.pull()
        if relaxed:
            _assert_relaxed_equal(ref, got, None, 0.0)
            ref.indirect[:, :] = got["indirect"]  # the next frame reads the lists in the order the device wrote them
        else:
            assert_world_equal(ref, got, what=f"{name} frame {f}")
    if slot:
        assert ctx.read_debug(False)[15] == 0, "alive bitmap and counters disagree"
    return got


def _edge_counts(k, chunks):
    sub, S = 32 * k, 32 * k * chunks
    return sorted({sub - 1, sub + 1, S - 1, S, S + 1, 2 * S + 1})


def _tile_edges(ctx, orc, name, **mode):
    """One instance per alive count at the edges of a sub-tile (sub = 32 K rows) and of a tile (S rows), each in a batch of
    its own: a burst of exactly that count, frames in which it dies off, then a burst into the shuffled dead stack."""
    k = tile_k(EFFECTS[name][1])
    counts = _edge_counts(k, ctx.tile_chunks)
    ref = _world(name, [n + 96 for n in counts], batches=[[i] for i in range(len(counts))], align=32)
    schedule = [counts] + [[0] * len(counts)] * 6 + [[80] * len(counts), [0] * len(counts)]
    _run(ctx, orc, name, ref, schedule, **mode)
    assert all(ref.metadata[i].particle_counter == n + 80 for i, n in enumerate(counts)), "every burst found free slots"
    assert all(ref.metadata[i].alive_count < n for i, n in enumerate(counts) if n > 80), "the frames had deaths"


@pytest.mark.parametrize("shaped_ctx,name", _shapes(ALL), indirect=["shaped_ctx"])
def test_tile_edges(shaped_ctx, orc, name):
    _tile_edges(shaped_ctx, orc, name)


@pytest.mark.parametrize("shaped_ctx,name", _shapes(ALL), indirect=["shaped_ctx"])
def test_many_instances_one_batch(shaped_ctx, orc, name):
    """Capacities off the tile grid, one instance that never spawns, per-instance properties, seeds and translations: the
    per-tile instance lookup and Properties staging switch instances inside a warp's run of tiles."""
    k = tile_k(EFFECTS[name][1])
    S = 32 * k * shaped_ctx.tile_chunks
    caps = [2 * S + 37, 19, 3 * 32 * k + 5, 40, S - 7, S + 90]
    ref = _world(name, caps)
    rng = np.random.default_rng(S + k)
    schedule = [[c if i != 3 else 0 for i, c in enumerate(caps)]]
    schedule += [[int(x) if i != 3 else 0 for i, x in enumerate(rng.integers(0, S // 3 + 2, len(caps)))] for _ in range(7)]
    _run(shaped_ctx, orc, name, ref, schedule)
    assert ref.metadata[3].particle_counter == 0 and ref.metadata[0].particle_counter > caps[0]


@pytest.mark.parametrize("shaped_ctx,name", _shapes(SECTOR), indirect=["shaped_ctx"])
def test_sector_planes(shaped_ctx, orc, name):
    _tile_edges(shaped_ctx, orc, name, sector=True)


@pytest.mark.parametrize("shaped_ctx,name", _shapes(["trails48", "vec4x4_96"]), indirect=["shaped_ctx"])
def test_slot_order(shaped_ctx, orc, name):
    """Instances on multiples of 32 rows; a lane owns bitmap word j*K + k of the tile, for chunks x K words."""
    _tile_edges(shaped_ctx, orc, name, slot=True)


@pytest.mark.parametrize("shaped_ctx,name", [pytest.param(8, "trails48", id="trails48-8sub"), pytest.param(16, "vec4x4_96", id="vec4x4_96-16sub")],
                         indirect=["shaped_ctx"])
def test_relaxed_order(shaped_ctx, orc, name):
    """Lists and dead stacks compared as sets (their order depends on scheduling), counts and particles exactly."""
    _tile_edges(shaped_ctx, orc, name, relaxed=True)


# ---- the slab-size rule ------------------------------------------------------------------------------------------------
# The update kernel's dynamic shared memory (42.5 KiB at the default rows per lane) leaves room for at most 5
# CTAs of 8 warps on an H100's 228 KiB: from 8 waves of those warps up, plan_batch always picks the largest tile.
MAX_CTAS_PER_SM = 5


@pytest.mark.parametrize("name", ["trails48", "vec4x4_96"])
def test_slab_size_rule_picks_the_largest_tile(native, orc, monkeypatch, name):
    import torch
    monkeypatch.delenv("HNB_TILE_CHUNKS", raising=False)
    monkeypatch.delenv("HNB_TILE_K", raising=False)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    k = tile_k(EFFECTS[name][1])
    warps = MAX_CTAS_PER_SM * sms * 8
    rows = 8 * warps * 32 * k
    print(f"{name}: K = {k}, {rows} rows = 8 waves of {warps} warps (at most {MAX_CTAS_PER_SM} CTAs on each of {sms} SMs)")
    ref = _world(name, [rows])
    c = native.Context(0)
    try:
        _run(c, orc, name, ref, [[rows - 1000], [0], [0], [900]])
        assert c.read_tile_size(0) == 32 * k * (ROWS_PER_LANE // k)
    finally:
        c.close()


# ---- C5 with K forced: 16, 8 and 2 sub-tiles per tile at most ----------------------------------------------------------
C5_FORCED = [(1, 16), (2, 8), (8, 2)]  # (K, the largest sub-tile count)


@pytest.mark.parametrize("shaped_ctx", [(n, k) for k, n in C5_FORCED], ids=[f"K{k}-{n}sub" for k, n in C5_FORCED], indirect=True)
@pytest.mark.parametrize("end", ["sub-1", "sub+1", "S-1", "S+1"])
def test_c5_claim_ending_at_tile_edges(shaped_ctx, orc, end):
    """tests/test_gpu_identity_claim.py's claim-edge scenario, with the claim ending next to a sub-tile or tile edge of
    the forced shape: the tile_known shortcut and the claimed prefetch over up to 16 sub-tiles."""
    ctx = shaped_ctx
    ctx.stride = 32
    sub = 32 * ctx.forced_k
    S = sub * ctx.tile_chunks
    L, cap = {"sub-1": sub - 1, "sub+1": sub + 1, "S-1": S - 1, "S+1": S + 1}[end], 4096
    ref = claim_edge_world(L, cap)
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    ctx.slab_fill_c5(gpu.slab, 0, cap, 1, 1e9, 1e9)
    ctx.slab_upload_aos(gpu.slab, 0, ref.particles)
    _frames(orc, ref, gpu, [[s] for s in CLAIM_EDGE_SPAWNS], f"claim ending at row {L}")
    assert ref.metadata[0].alive_count == 1000


@pytest.mark.parametrize("shaped_ctx", [(16, 1)], ids=["K1-16sub"], indirect=True)
def test_c5_claimed_entries_are_neither_loaded_nor_stored(shaped_ctx, orc):
    shaped_ctx.stride = 32
    claims.test_claimed_entries_are_neither_loaded_nor_stored(shaped_ctx, orc)


@pytest.mark.parametrize("shaped_ctx", [(16, 1)], ids=["K1-16sub"], indirect=True)
def test_ordered_events_parent_at_16_sub_tiles(shaped_ctx, orc):
    """The ordered-events scenario with every effect at K = 1: the parent's event rows row0 + (j*K + k)*32 + lane."""
    shaped_ctx.stride = 32
    ordered_events.test_ordered_events_two_children(shaped_ctx, orc, 6000)
    shaped_ctx.batches = [shaped_ctx.tile_batch]


# ---- rows per lane -----------------------------------------------------------------------------------------------------
def test_rows_per_lane_above_32_is_clamped(native, orc, monkeypatch):
    """HNB_ROWS_PER_LANE = 64 runs as 32: with 8 forced sub-tiles C5's 1024-row tiles span exactly 32 bitmap words, one per
    lane, in slot order (beyond 32 words lanes would wrap)."""
    monkeypatch.setenv("HNB_ROWS_PER_LANE", "64")
    monkeypatch.setenv("HNB_TILE_CHUNKS", "16")  # clamped to 32 / 4 = 8
    monkeypatch.delenv("HNB_TILE_K", raising=False)
    c = native.Context(0)
    try:
        rng = np.random.default_rng(64)
        ref = RefWorld(6000, 8, [Instance(0, 6000, alive=5000, seed=42)])
        _fill(ref, rng, 0.02, 0.3)
        _run_c5(c, orc, ref, 16)
        assert c.read_tile_size(0) == 32 * 32
    finally:
        c.close()
