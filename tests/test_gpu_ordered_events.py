"""HNB_EFFECT_ORDERED_EVENTS on the device."""
from collections import Counter  # noqa: F401

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import runtime as R
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.helpers import Instance, RefWorld, at_tile_sizes, tiled_ctx  # noqa: F401
from tests.test_gpu_events import EVENT_CAP, _oracle_append_events, _oracle_child_init

pytestmark = pytest.mark.gpu
A = G.Attribute


@at_tile_sizes("pcap", [1024, 6000])
def test_ordered_events_two_children(tiled_ctx, orc, pcap):
    """HNB_EFFECT_ORDERED_EVENTS on the device : with
    ordered append the buffers must hold EXACTLY the canonical sequence, overflow included, and the children need no
    re-ordering of the oracle's events. With the slab-size rule and at 2-4 forced sub-tiles per tile: an event's row is row0 + (j*K + k)*32 + lane. Scenario: one parent, two event channels: channel 0 fed every frame by particles that are alive (EventEmitCondition::Always,
    count 0 or 1 drawn per particle), channel 1 by dying particles (OnDie, 4 events each). Each child consumes its
    own buffer the frame after. Children come BEFORE the parent in batch order, as EffectSorter places them
    (batch.rs:599-603), so a child's init reads the parent's records before the parent's init recycles slots."""
    wp = G.ExprWriter()
    parent = (G.EffectAsset(pcap, wp.module, name="emitter")
              .init(G.SetAttributeModifier(A.POSITION, wp.rand(G.VEC3) * wp.lit(2.) - wp.lit(1.)))
              .init(G.SetAttributeModifier(A.VELOCITY, wp.rand(G.VEC3) - wp.lit(0.5)))
              .init(G.SetAttributeModifier(A.AGE, wp.lit(0.)))
              .init(G.SetAttributeModifier(A.LIFETIME, wp.lit(0.1).uniform(wp.lit(0.5))))
              .update(G.EmitSpawnEventModifier(G.ALWAYS, (wp.rand(G.FLOAT) * wp.lit(1.25)).cast(G.UINT), 0))
              .update(G.EmitSpawnEventModifier(G.ON_DIE, wp.lit(G.U32(4)), 1)))
    children = []
    for tag in (0, 1):
        wc = G.ExprWriter()
        children.append(G.EffectAsset(4096, wc.module, name=f"child{tag}")
                        .init(G.InheritAttributeModifier(A.POSITION))
                        .init(G.SetAttributeModifier(A.VELOCITY, wc.parent_attr(A.VELOCITY) * wc.lit(0.25 + tag) + (wc.rand(G.VEC3) - wc.lit(0.5))))
                        .init(G.SetAttributeModifier(A.AGE, wc.lit(0.)))
                        .init(G.SetAttributeModifier(A.LIFETIME, wc.lit(0.2 + 0.1 * tag)))
                        .init(G.SetAttributeModifier(A.U32_0, wc.parent_attr(A.ID))))
    p_fx = parent.generate(num_event_bindings=2, ordered_events=True)
    c_fx = [c.generate(parent=parent) for c in children]
    p_stride, c_stride = p_fx.particle_stride, c_fx[0].particle_stride
    dt = 1.0 / 30.0
    ctx = tiled_ctx
    ctx.tile_batch = 2  # the parent: 32-byte records, 128-row sub-tiles (the children's 48-byte records have 64-row ones)
    pw = RefWorld(pcap, p_stride // 4, [Instance(0, pcap, alive=0, seed=1)], dt=dt)
    cw = [RefWorld(4096, c_stride // 4, [Instance(0, 4096, alive=0, seed=2 + k)], dt=dt) for k in (0, 1)]
    po, co = EffectOracle(parent), [EffectOracle(c) for c in children]
    events = [np.zeros(EVENT_CAP, dtype=np.uint32) for _ in (0, 1)]
    event_count = [0, 0]

    # GPU tables: rows 0, 1 = children (batches 0, 1), row 2 = parent (batch 2); child infos 0, 1 = channels 0, 1
    p_slab = ctx.slab_create(pcap, p_stride)
    c_slab = [ctx.slab_create(4096, c_stride) for _ in (0, 1)]
    p_eff = ctx.effect_compile(p_fx)
    c_eff = [ctx.effect_compile(fx) for fx in c_fx]
    evbuf = [ctx.event_buffer_create(EVENT_CAP) for _ in (0, 1)]
    for k in (0, 1):
        ctx.child_info_insert(k, 0, 0)
        md_c = R.initial_metadata(4096, k, c_stride // 4)
        md_c.global_child_index, md_c.local_child_index = k, k
        ctx.metadata_insert(k, md_c)
        ctx.draw_args_insert(k)
    md_p = R.initial_metadata(pcap, 2, p_stride // 4)
    md_p.base_child_index = 0
    ctx.metadata_insert(2, md_p)
    ctx.draw_args_insert(2)

    spawn_sched = [s * pcap // 1024 for s in [700, 0, 0, 150, 0, 0, 0, 800, 0, 0, 0, 0, 100, 0, 0, 0, 0, 0, 0, 0]]
    spawned = [0, 0]
    overflowed = False
    seen_counts = []
    all_emitted = [[], []]
    for f, spawn in enumerate(spawn_sched):
        seed_p = int(pcg_hash(np.array([5000 + f], dtype=np.uint32))[0])
        seed_c = [int(pcg_hash(np.array([6000 + 10 * f + k], dtype=np.uint32))[0]) for k in (0, 1)]
        ctx.upload_spawners([R.make_spawner(spawn=0, seed=seed_c[k], effect_metadata_index=k, draw_indirect_index=k, slab_offset=0, parent_slab_offset=0)
                             for k in (0, 1)]
                            + [R.make_spawner(spawn=spawn, seed=seed_p, effect_metadata_index=2, draw_indirect_index=2, slab_offset=0)])
        ctx.upload_batches([N.BatchInfo(0, 0, 0, 0, 0, 1), N.BatchInfo(0, 0, 1, 0, 1, 1), N.BatchInfo(0, 0, 2, 0, 2, 1)], [0, 0, 0])
        ctx.set_sim_params(dt, f * dt, 3)
        # what the previous frame's update left in the two buffers
        n_valid = []
        for k in (0, 1):
            assert ctx.read_child_info(k).event_count == event_count[k], f"frame {f} channel {k}"
            nv = min(event_count[k], EVENT_CAP)
            overflowed |= event_count[k] > EVENT_CAP
            seen_counts.append(event_count[k])
            got = ctx.event_buffer_download(evbuf[k], 0, EVENT_CAP)
            np.testing.assert_array_equal(got[:nv], events[k][:nv], err_msg=f"frame {f} channel {k}: event order")
            n_valid.append(nv)
        ctx.simulate([N.BatchLaunch.make(c_eff[0], c_slab[0], 0, 0, parent_slab=p_slab, consume_events=evbuf[0]),
                      N.BatchLaunch.make(c_eff[1], c_slab[1], 1, 0, parent_slab=p_slab, consume_events=evbuf[1]),
                      N.BatchLaunch.make(p_eff, p_slab, 2, spawn, emit_events=evbuf)])

        # ----- oracle frame: inits (children read the parent's records as the previous frame left them), ...
        t = np.float32(f * dt)
        pw.sim.time = t
        for k in (0, 1):
            cw[k].sim.time = t
            cw[k].set_spawns([0], [seed_c[k]])
            spawned[k] += _oracle_child_init(children[k], co[k], cw[k], po, pw, events[k], n_valid[k], seed_c[k])
        pw.set_spawns([spawn], [seed_p])
        po.init_pass(pw)
        # ... indirect (clears the event counts, vfx_indirect.wgsl:38-46) + prefix sums, updates, event appends
        event_count = [0, 0]
        for w in (cw[0], cw[1], pw):
            w.oracle_indirect(orc)
            w.oracle_prefix_sum(orc)
        for k in (0, 1):
            co[k].update_pass(cw[k])
        po.update_pass(pw)
        assert [ch for ch, _ in po.last_emitted] == [0, 1]
        for channel, counts in po.last_emitted:
            event_count[channel] = _oracle_append_events(pw, counts, events[channel], event_count[channel])
            rows_read = pw.indirect[:pw.metadata[0].max_update, 1 - pw.metadata[0].indirect_write_index]
            all_emitted[channel] = np.repeat(rows_read, counts[:len(rows_read)]).tolist()

        # ----- compare
        ctx.sync()
        for world, slab, row, stride, rows in ((cw[0], c_slab[0], 0, c_stride, 4096), (cw[1], c_slab[1], 1, c_stride, 4096), (pw, p_slab, 2, p_stride, pcap)):
            m_gpu = np.frombuffer(bytes(ctx.read_metadata(row)), dtype=np.uint32)
            m_ref = world.metadata_rows()[0].copy()
            m_ref[5] = row
            for fld in (7, 8, 9, 10):
                m_ref[fld] = m_gpu[fld]
            np.testing.assert_array_equal(m_gpu, m_ref, err_msg=f"frame {f} metadata row {row}")
            assert ctx.read_draw_args(row).instance_count == world.draw[1]
            np.testing.assert_array_equal(ctx.slab_download_indirect(slab, 0, rows), world.indirect, err_msg=f"frame {f} row {row}: lists")
            np.testing.assert_array_equal(ctx.slab_download_aos(slab, 0, rows, stride), world.particles, err_msg=f"frame {f} row {row}: particles")
    assert spawned[0] > 100 and spawned[1] > 100, spawned
    assert overflowed and min(seen_counts[2:]) < EVENT_CAP, f"the scenario must both overflow an event buffer (capped appends) and not: {seen_counts}"
