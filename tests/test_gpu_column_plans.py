"""Column plans on the device: a C5 slab whose update leaves lifetime alone stores three of its four columns, and every
state it reaches is the state of the same instance on a slab in the default cut, bit for bit."""
import numpy as np
import pytest

from tests.helpers import Lockstep, sparks_world

pytestmark = pytest.mark.gpu

C5_PLAN = [(0, 16), (16, 8), (24, 4), (28, 4)]
DEFAULT_CUT = [(0, 16), (16, 16)]
P = 1 << 20


def _plan(ctx, slab):
    v = ctx.slab_device_view(slab)
    return [(v.plane_offset[p], v.plane_width[p]) for p in range(v.num_planes)], v


def _c5_pair(ctx, lo, hi):
    """The same filled C5 instance on two slabs: slab 0 runs the authored C5 (lifetime read-only), whose first launch moves
    the filled records into its plan; slab 1 runs the hand-lowered C5, which writes every word (the default cut). Metadata
    rows 0 and 1, one batch each."""
    from bevy_hanabi_b200 import _native as N, recipes, runtime as R
    effects = [ctx.effect_compile(recipes.c5_asset(P).generate()), ctx.effect_compile(recipes.c5_lowered())]
    slabs = [ctx.slab_create(P, 32) for _ in range(2)]
    for s in slabs:  # no device view before the first launch: a view pins the plan it shows
        ctx.slab_fill_c5(s, 0, P, 77, lo, hi)
    for i in range(2):
        md = R.initial_metadata(P, i, 8)
        md.alive_count, md.max_spawn = P, 0
        ctx.metadata_insert(i, md)
        ctx.draw_args_insert(i, N.DrawIndexedIndirectArgs(0, 0, 0, 0, 0))
    ctx.upload_spawners([R.make_spawner(seed=42, effect_metadata_index=i, draw_indirect_index=i) for i in range(2)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1), N.BatchInfo(0, 0, 1, 0, 1, 1)], [0, 0])
    ctx.set_sim_params(1.0 / 60.0, 0.0, 2)
    launches = [N.BatchLaunch.make(effects[i], slabs[i], i, 0) for i in range(2)]
    ctx.simulate(launches)
    assert _plan(ctx, slabs[0])[0] == C5_PLAN and _plan(ctx, slabs[1])[0] == DEFAULT_CUT
    return effects, slabs, launches


def _same(ctx, slabs, what):
    assert ctx.slab_checksum(slabs[0], 0, P) == ctx.slab_checksum(slabs[1], 0, P), what
    assert ctx.slab_checksum_indirect(slabs[0], 0, P) == ctx.slab_checksum_indirect(slabs[1], 0, P), what
    a, b = ctx.read_metadata(0), ctx.read_metadata(1)
    assert (a.alive_count, a.max_spawn, a.indirect_write_index) == (b.alive_count, b.max_spawn, b.indirect_write_index), what


def test_c5_plan_equals_default_cut_for_120_frames(ctx):
    """Kills along the way (lifetimes 0.05 to 4 s over 2 s of frames); the lifetime column of the C5-plan slab never
    changes."""
    effects, slabs, launches = _c5_pair(ctx, 0.05, 4.0)
    _same(ctx, slabs, "frame 0")
    _, view = _plan(ctx, slabs[0])
    life_before = ctx.device_download(view.planes[3], 4 * P)
    for f in range(1, 121):
        ctx.simulate(launches)
        if f % 20 == 19:
            _same(ctx, slabs, f"frame {f}")
    alive = ctx.read_metadata(0).alive_count
    assert 0 < alive < P, "the scenario must kill some particles and keep some"
    np.testing.assert_array_equal(ctx.device_download(view.planes[3], 4 * P), life_before, err_msg="lifetime column")
    assert ctx.plan_compiles() == 0


def test_snapshot_restore_across_plans_and_repack(ctx):
    """Snapshot from either plan, restore into the other: both slabs stay equal, through a repack of both, and after the
    authored effect takes over the default-cut slab (a module compiled for that plan)."""
    from bevy_hanabi_b200 import _native as N
    effects, slabs, launches = _c5_pair(ctx, 0.05, 1.0)
    for _ in range(30):
        ctx.simulate(launches)
    _same(ctx, slabs, "before the snapshots")
    nbytes = ctx.instance_snapshot_bytes(32, P)
    bufs = [ctx.device_alloc(nbytes) for _ in range(2)]
    try:
        for i in range(2):
            ctx.instance_snapshot(slabs[i], effects[i], i, 0, P, bufs[i], nbytes)
        ctx.instance_restore(slabs[0], effects[0], 0, 0, P, bufs[1], nbytes)  # default cut -> C5 plan
        ctx.instance_restore(slabs[1], effects[1], 1, 0, P, bufs[0], nbytes)  # C5 plan -> default cut
        ctx.sync()
        _same(ctx, slabs, "after the crossed restores")
        for _ in range(10):
            ctx.simulate(launches)
        ctx.slab_repack(slabs[0], effects[0], 0, 0, P)
        ctx.slab_repack(slabs[1], effects[1], 1, 0, P)
        for _ in range(10):
            ctx.simulate(launches)
        _same(ctx, slabs, "after repack + 10 frames")
        assert ctx.plan_compiles() == 0
        launches[1] = N.BatchLaunch.make(effects[0], slabs[1], 1, 0)
        for _ in range(10):
            ctx.simulate(launches)
        _same(ctx, slabs, "the authored C5 on both slabs")
        assert ctx.plan_compiles() == 1
        assert _plan(ctx, slabs[0])[0] == C5_PLAN and _plan(ctx, slabs[1])[0] == DEFAULT_CUT
    finally:
        for b in bufs:
            ctx.device_free(b)


def test_init_spawned_effect_on_its_own_plan(ctx, orc):
    """An authored effect with read-only attributes, spawning into recycled slots of a slab its first launch gives its own
    plan, equals the interpreter every frame."""
    asset, ref = sparks_world([3000, 1000])
    lock = Lockstep(ctx, orc, ref, asset)
    plan = asset.generate().column_plan()
    assert plan != [(0, 16), (16, 16)], "the sparks must have read-only attributes"
    # the world was uploaded in the default cut; the first launch moves it into the effect's own plan
    lock.run([[120, 40]] * 12 + [[0, 0]] * 6 + [[200, 10]] * 12, what="own plan")
    assert _plan(ctx, lock.gpu.slab)[0] == plan
    assert ctx.plan_compiles() == 0


def test_view_taken_before_the_first_launch_stays_valid(ctx):
    """A device view of a filled slab, taken before any effect is bound, pins the default cut: the authored C5 then runs
    a module generated for that cut, and the view's columns still hold the records after the frames."""
    from bevy_hanabi_b200 import _native as N, recipes, runtime as R
    n = 1 << 16
    slab = ctx.slab_create(n, 32)
    ctx.slab_fill_c5(slab, 0, n, 5, 0.05, 1.0)
    plan, view = _plan(ctx, slab)
    assert plan == DEFAULT_CUT
    effect = ctx.effect_compile(recipes.c5_asset(n).generate())
    md = R.initial_metadata(n, 0, 8)
    md.alive_count, md.max_spawn = n, 0
    ctx.metadata_insert(0, md)
    ctx.draw_args_insert(0)
    ctx.upload_spawners([R.make_spawner(seed=42)])
    ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1)], [0])
    ctx.set_sim_params(1.0 / 60.0, 0.0, 1)
    for _ in range(20):
        ctx.simulate([N.BatchLaunch.make(effect, slab, 0, 0)])
    ctx.sync()
    assert _plan(ctx, slab)[0] == DEFAULT_CUT and ctx.plan_compiles() == 1
    cols = [ctx.device_download(view.planes[p], n * 16).reshape(n, 4) for p in range(2)]
    np.testing.assert_array_equal(np.concatenate(cols, axis=1), ctx.slab_download_aos(slab, 0, n, 32))
    assert 0 < ctx.read_metadata(0).alive_count < n
