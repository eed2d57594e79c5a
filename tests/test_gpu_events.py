"""GPU spawn events (SURVEY.md §8f-1): a parent effect emits events from its update pass
(EmitSpawnEventModifier, src/modifier/mod.rs:654-717; append_spawn_events_N, src/lib.rs:976-993), a child effect
consumes them in the NEXT frame's init pass (vfx_init.wgsl:123-129, :166-171) and inherits attributes from the
parent particle (InheritAttributeModifier, src/modifier/attr.rs:173-186).

Like in the reference, the ORDER in which events land in the buffer depends on atomic scheduling, so the event
buffer — and therefore which child slot receives which event — is compared as a multiset; counts are exact.
"""
import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import runtime as R
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.effects import EVENT_CAP, event_assets
from tests.helpers import Instance, RefWorld, emitter_scene, oracle_append_events, oracle_child_init

pytestmark = pytest.mark.gpu


def _sorted_rows(a):
    return a[np.lexsort(a.T[::-1])]


def test_parent_emits_child_consumes(ctx, orc):
    parent, child = event_assets()
    p_fx = parent.generate(num_event_bindings=1)
    c_fx = child.generate(parent=parent)
    assert p_fx.flags & N.EFFECT_EMIT_GPU_SPAWN_EVENTS
    assert c_fx.flags & N.EFFECT_CONSUME_GPU_SPAWN_EVENTS and c_fx.flags & N.EFFECT_READ_PARENT_PARTICLE
    p_stride, c_stride = p_fx.particle_stride, c_fx.particle_stride
    dt = 1.0 / 30.0

    # ---- oracle worlds (one slab each) and oracles
    pw = RefWorld(512, p_stride // 4, [Instance(0, 512, alive=0, seed=11)], dt=dt)
    cw = RefWorld(2048, c_stride // 4, [Instance(0, 2048, alive=0, seed=22)], dt=dt)
    po, co = EffectOracle(parent), EffectOracle(child)
    events = np.zeros(EVENT_CAP, dtype=np.uint32)
    event_count = 0

    # ---- GPU: one context, two slabs, spawner/metadata rows 0 (parent) and 1 (child), two batches
    p_slab, c_slab = ctx.slab_create(512, p_stride), ctx.slab_create(2048, c_stride)
    p_eff, c_eff = ctx.effect_compile(p_fx), ctx.effect_compile(c_fx)
    evbuf = ctx.event_buffer_create(EVENT_CAP)
    ctx.child_info_insert(0, 0, 0)
    md_p = R.initial_metadata(512, 0, p_stride // 4)
    md_p.base_child_index = 0
    md_c = R.initial_metadata(2048, 1, c_stride // 4)
    md_c.global_child_index = 0
    md_c.local_child_index = 0
    ctx.metadata_insert(0, md_p)
    ctx.metadata_insert(1, md_c)
    ctx.draw_args_insert(0)
    ctx.draw_args_insert(1)
    launches = [N.BatchLaunch.make(p_eff, p_slab, 0, 0, emit_events=[evbuf]),
                N.BatchLaunch.make(c_eff, c_slab, 1, 0, parent_slab=p_slab, consume_events=evbuf)]

    spawn_sched = [40, 0, 25, 0, 0, 60, 0, 0, 10, 0, 0, 0, 30, 0, 0, 0, 0, 0]
    total_child_spawned = 0
    for f, spawn in enumerate(spawn_sched):
        seed_p = int(pcg_hash(np.array([100 + f], dtype=np.uint32))[0])
        seed_c = int(pcg_hash(np.array([900 + f], dtype=np.uint32))[0])
        # ----- GPU frame
        ctx.upload_spawners([R.make_spawner(spawn=spawn, seed=seed_p, effect_metadata_index=0, draw_indirect_index=0, slab_offset=0),
                             R.make_spawner(spawn=0, seed=seed_c, effect_metadata_index=1, draw_indirect_index=1, slab_offset=0,
                                            parent_slab_offset=0)])
        ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1), N.BatchInfo(0, 0, 1, 0, 1, 1)], [0, 0])
        ctx.set_sim_params(dt, f * dt, 2)
        launches[0] = N.BatchLaunch.make(p_eff, p_slab, 0, spawn, emit_events=[evbuf])
        # events written by the previous frame's update, as the child's init is about to see them
        gpu_event_count = ctx.read_child_info(0).event_count
        gpu_events = ctx.event_buffer_download(evbuf, 0, EVENT_CAP)
        assert gpu_event_count == event_count
        n_valid = min(event_count, EVENT_CAP)
        assert sorted(gpu_events[:n_valid].tolist()) == sorted(events[:n_valid].tolist())
        # make the oracle consume the events in the order the GPU buffer holds them (reference order is unspecified)
        events[:n_valid] = gpu_events[:n_valid]
        ctx.simulate(launches)

        # ----- oracle frame
        pw.sim.time = cw.sim.time = np.float32(f * dt)
        pw.set_spawns([spawn], [seed_p])
        cw.set_spawns([0], [seed_c])
        po.init_pass(pw)
        total_child_spawned += oracle_child_init(child, co, cw, po, pw, events, n_valid, seed_c)
        # indirect + prefix for both worlds, events cleared (vfx_indirect.wgsl:38-46)
        event_count = 0
        for w in (pw, cw):
            w.oracle_indirect(orc)
            w.oracle_prefix_sum(orc)
        po.update_pass(pw)
        co.update_pass(cw)
        for channel, counts in po.last_emitted:
            assert channel == 0
            event_count = oracle_append_events(pw, counts, events, event_count)

        # ----- compare
        ctx.sync()
        for world, slab, row, stride in ((pw, p_slab, 0, p_stride), (cw, c_slab, 1, c_stride)):
            m_gpu = np.frombuffer(bytes(ctx.read_metadata(row)), dtype=np.uint32)
            m_ref = world.metadata_rows()[0].copy()
            m_ref[5] = row  # indirect_draw_index differs between the single-instance oracle worlds and the shared GPU tables
            for fld in (7, 8, 9, 10):
                m_ref[fld] = m_gpu[fld]
            np.testing.assert_array_equal(m_gpu, m_ref, err_msg=f"frame {f} metadata row {row}")
            assert ctx.read_draw_args(row).instance_count == world.draw[1]
        # parent: fully deterministic -> exact
        np.testing.assert_array_equal(ctx.slab_download_aos(p_slab, 0, 512, p_stride), pw.particles)
        np.testing.assert_array_equal(ctx.slab_download_indirect(p_slab, 0, 512), pw.indirect)
        # child: exact as well, because the oracle consumed the events in the GPU buffer's order
        np.testing.assert_array_equal(ctx.slab_download_aos(c_slab, 0, 2048, c_stride), cw.particles)
        np.testing.assert_array_equal(ctx.slab_download_indirect(c_slab, 0, 2048), cw.indirect)
    assert total_child_spawned > 100, "the scenario must actually spawn children from events"
    assert event_count >= 0


def test_two_children_two_conditions(ctx, orc):
    """One parent, two event channels: channel 0 fed every frame by particles that are alive (EventEmitCondition::Always,
    count 0 or 1 drawn per particle), channel 1 by dying particles (OnDie, 4 events each). Each child consumes its
    own buffer the frame after. Children come BEFORE the parent in batch order, as EffectSorter places them
    (batch.rs:599-603), so a child's init reads the parent's records before the parent's init recycles slots."""
    emitter_scene(ctx, orc, 1024, ordered=False)
