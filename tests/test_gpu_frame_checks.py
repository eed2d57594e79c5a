"""A frame hnb_simulate refuses leaves no trace: every launch is checked before the context writes its host frame block,
clears or grows tile states, or enqueues anything. After each refused frame the tile-size words of every batch row, the
tile-state clear count, the epoch, the launch count and the metadata rows are as they were; the corrected frame then runs
against the oracle and clears the tile states of each slot-order batch slot it uses for the first time exactly once."""
import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from tests.effects import fill_c5, table_asset, table_props
from tests.helpers import Instance, Lockstep, RefWorld, seeds, table_world

pytestmark = pytest.mark.gpu


def _state(ctx, ref):
    n, nb = len(ref.instances), len(ref.batches)
    return dict(tile_sizes=[ctx.read_tile_size(b) for b in range(nb)], clears=ctx.tile_state_clears(), epoch=ctx.last_epoch(),
                launches=ctx.launch_count, metadata=[bytes(ctx.read_metadata(i)) for i in range(n)])


def _refused(ctx, ref, launches, code):
    """Runs the frame `launches`, which must fail with `code`, and checks that it changed nothing."""
    ctx.sync()
    before = _state(ctx, ref)
    with pytest.raises(N.HanabiError) as e:
        ctx.simulate(launches)
    assert e.value.code == code, e.value.message
    ctx.sync()
    assert _state(ctx, ref) == before, "a refused frame must leave the context as it was"
    return before["clears"]


def _two_slot_order_c5_batches(ctx, orc):
    ref = RefWorld(2048, 8, [Instance(0, 1024, alive=900, seed=1), Instance(1024, 1024, alive=500, seed=2)], batches=[[0], [1]])
    fill_c5(ref, np.random.default_rng(5), 0.02, 0.3)
    return ref, Lockstep(ctx, orc, ref, slot=True)


def test_missing_properties(ctx, orc):
    """A slot-order effect with a property, on a fresh batch slot, before its properties were uploaded."""
    ref = table_world("vec4x2_64", [256], align=32)
    asset = table_asset("vec4x2_64", 256)
    lock = Lockstep(ctx, orc, ref, asset, props=table_props("vec4x2_64", 1), slot=True, seeds=seeds)
    bare = ctx.effect_compile(asset.generate(slot_order=True))  # the same effect, no property record uploaded
    clears = _refused(ctx, ref, [N.BatchLaunch.make(bare, lock.gpu.slab, 0, 150)], N.HNB_ERR_NOT_READY)
    lock.run([[150]])
    assert ctx.tile_state_clears() == clears + 1
    lock.run([[40], [0], [0]], start=1)


def test_invalid_emit_buffer_after_a_slot_order_batch(ctx, orc):
    """Batch 0 is slot-order C5; batch 1 names an event buffer that does not exist."""
    ref, lock = _two_slot_order_c5_batches(ctx, orc)
    good = lock.gpu.launches()
    bad = N.BatchLaunch.make(lock.gpu.effect, lock.gpu.slab, 1, 0, emit_events=[99])
    clears = _refused(ctx, ref, [good[0], bad], N.HNB_ERR_INVALID_ARG)
    lock.run(1)
    assert ctx.tile_state_clears() == clears + 2
    lock.run(3, start=1)


def test_overlapping_slot_order_batches(ctx, orc):
    """Two slot-order batches that both claim instance 0."""
    ref, lock = _two_slot_order_c5_batches(ctx, orc)
    overlap = (N.BatchInfo * 2).from_buffer_copy(bytes(ref.batch_infos[0]) * 2)
    ctx.upload_batches_raw(overlap, 2, (N.u32 * 2)(0, 0), 2)
    clears = _refused(ctx, ref, lock.gpu.launches(), N.HNB_ERR_BATCH_COVERAGE)
    lock.run(1)  # uploads the batch table of the world again
    assert ctx.tile_state_clears() == clears + 2
    lock.run(3, start=1)
