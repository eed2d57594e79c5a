"""The real kernel templates (hnb_init / hnb_update of hnb_particle_kernels.cuh) executed on the CPU under the thread
emulation of tests/kernel_emu.py, against the oracle: alive lists in canonical order, dead stack, counters,
draw-indirect counts and every particle word, bit for bit — the same bar as the GPU suite, on small worlds."""
import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import recipes
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.helpers import Instance, RefWorld
from tests.kernel_emu import EmuWorld, tile_count
from tests.test_gpu_effects import _firework_trails
from tests.test_gpu_scene import _drifting_sparks

A = G.Attribute
pytestmark = pytest.mark.timeout(600)  # real threads: a protocol bug must fail, not hang


def _assert_same(ref, got, what):
    np.testing.assert_array_equal(got["metadata"], ref.metadata_rows(), err_msg=f"{what}: metadata")
    np.testing.assert_array_equal(got["draw"], ref.draw, err_msg=f"{what}: draw args")
    np.testing.assert_array_equal(got["prefix"], ref.prefix, err_msg=f"{what}: prefix sums")
    assert got["total_update"] == ref.batch_infos[0].total_update_count
    np.testing.assert_array_equal(got["indirect"], ref.indirect, err_msg=f"{what}: ping / pong / dead")
    np.testing.assert_array_equal(got["particles"], ref.particles, err_msg=f"{what}: particles")


def _c5_world(rng, insts):
    ref = RefWorld(sum(i.capacity for i in insts), 8, insts)
    for inst in ref.instances:
        n = inst.alive
        p = np.zeros((n, 8), dtype=np.float32)
        p[:, 0:3] = rng.uniform(-1, 1, (n, 3)); p[:, 4:7] = rng.uniform(-1, 1, (n, 3)); p[:, 7] = rng.uniform(0.02, 0.15, n)
        ref.particles[inst.slab_offset:inst.slab_offset + n] = p.view(np.uint32)
    return ref


@pytest.mark.parametrize("chunks,ctas", [(1, 1), (1, 3), (2, 2), (3, 2), (4, 2)])
def test_update_kernel_c5_single_instance(orc, chunks, ctas):
    """Tile tickets, look-back across 10-40 tiles, deferred compaction, dead-stack pushes, last-tile totals."""
    rng = np.random.default_rng(chunks * 10 + ctas)
    ref = _c5_world(rng, [Instance(0, 5000, alive=4700, seed=42)])
    emu = EmuWorld(ref, recipes.c5_lowered(), chunks=chunks, update_ctas=ctas)
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    for step in range(5):
        ref.oracle_frame(orc, orc.orc_body_update_c5(), k)
        emu.frame_step(orc, ref.sim, [0], [42])
        _assert_same(ref, emu.pull(), f"step {step}")
    assert 0 < ref.metadata[0].alive_count < 4700


def test_update_kernel_many_instances_one_batch(orc):
    """Instances smaller than, equal to and larger than a tile, empty ones, in one launch: per-tile instance lookup,
    one look-back chain per instance."""
    rng = np.random.default_rng(3)
    caps = [40, 128, 129, 700, 1, 256, 90, 1500]
    alive = [40, 128, 100, 650, 0, 256, 0, 1400]
    insts, off = [], 0
    for c, a in zip(caps, alive):
        insts.append(Instance(off, c, alive=a, seed=off + 5))
        off += c
    ref = _c5_world(rng, insts)
    emu = EmuWorld(ref, recipes.c5_lowered(), chunks=1, update_ctas=2)
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    seeds = [i.seed for i in insts]
    for step in range(4):
        ref.oracle_frame(orc, orc.orc_body_update_c5(), k)
        emu.frame_step(orc, ref.sim, [0] * len(insts), seeds)
        _assert_same(ref, emu.pull(), f"step {step}")


@pytest.mark.parametrize("name", ["trails", "sparks"])
def test_init_and_update_kernels_authored_effects(orc, name):
    """Bursts into recycled slots: rank-based dead-slot pops of hnb_init (4 spawns per thread), spawn caps, then the
    update kernel on the grown lists — against the numpy interpreter of the same effect."""
    asset = {"trails": _firework_trails, "sparks": _drifting_sparks}[name](1500)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(1500, size // 4, [Instance(0, 1500, alive=0, seed=1)], dt=1.0 / 10.0)
    eo = EffectOracle(asset)
    emu = EmuWorld(ref, asset.generate(), chunks=1, update_ctas=2)
    recycled = False
    for f in range(7):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawn = [900 if f % 3 == 0 else 37]
        seed = [int(pcg_hash(np.array([0x1234 + f], dtype=np.uint32))[0])]
        ref.set_spawns(spawn, seed)
        before = ref.metadata[0].particle_counter
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawn, seed)
        _assert_same(ref, emu.pull(), f"frame {f}")
        recycled |= ref.metadata[0].particle_counter - before < spawn[0] or ref.metadata[0].particle_counter > 1500
    assert recycled, "the scenario must hit the spawn cap or reuse freed slots"


def test_update_kernel_more_instances_than_the_shared_table(orc):
    """2500 instances in one batch: the tile-prefix table is searched in global memory (n_effects > 2047)."""
    rng = np.random.default_rng(8)
    caps = rng.integers(1, 12, 2500)
    insts, off = [], 0
    for c in caps:
        a = int(rng.integers(0, c + 1)) if rng.random() > 0.15 else 0
        insts.append(Instance(off, int(c), alive=a, seed=off * 7 + 1))
        off += int(c)
    ref = _c5_world(rng, insts)
    emu = EmuWorld(ref, recipes.c5_lowered(), chunks=1, update_ctas=2)
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    seeds = [i.seed for i in insts]
    for step in range(3):
        ref.oracle_frame(orc, orc.orc_body_update_c5(), k)
        emu.frame_step(orc, ref.sim, [0] * len(insts), seeds)
        _assert_same(ref, emu.pull(), f"step {step}")


def test_relaxed_order_variant_same_sets(orc):
    """HNB_EFFECT_RELAXED_ORDER: one warp-aggregated atomic per tile instead of the look-back chain — list ORDER is
    scheduling-dependent (like the reference's), counts, sets and particle words are not."""
    rng = np.random.default_rng(4)
    ref = _c5_world(rng, [Instance(0, 3000, alive=2800, seed=9)])
    emu = EmuWorld(ref, recipes.c5_lowered(relaxed_order=True), chunks=2, update_ctas=2)
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    for step in range(4):
        ref.oracle_frame(orc, orc.orc_body_update_c5(), k)
        emu.frame_step(orc, ref.sim, [0], [9])
        got = emu.pull()
        np.testing.assert_array_equal(got["metadata"], ref.metadata_rows())
        np.testing.assert_array_equal(got["draw"], ref.draw)
        np.testing.assert_array_equal(got["particles"], ref.particles)
        md = ref.metadata[0]
        W, alive = md.indirect_write_index, md.alive_count
        assert sorted(got["indirect"][:alive, W].tolist()) == sorted(ref.indirect[:alive, W].tolist())
        assert sorted(got["indirect"][alive:3000, 2].tolist()) == sorted(ref.indirect[alive:3000, 2].tolist())
        # the next frame reads the list the emulated kernel wrote: keep the oracle on the same order
        ref.indirect[:, :] = got["indirect"]


def test_kernels_with_properties_and_transcendentals(orc):
    """C3 force field: per-instance Properties staged by the update kernel, sphere sampling in init. libm on the host
    vs numpy: 1e-5 of the attribute's magnitude per step, integer structures exact."""
    from tests.helpers import assert_float_attributes_close
    from tests.test_gpu_effects import _float_word_mask, _force_field
    asset = _force_field(2048)
    _, size, _ = asset.particle_layout()
    props = {"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}
    ref = RefWorld(2048, size // 4, [Instance(0, 2048, alive=0, seed=77)])
    ref.metadata[0].properties_array_index = 0
    eo = EffectOracle(asset, {0: props})
    emu = EmuWorld(ref, asset.generate(), chunks=1, update_ctas=2, property_blobs=[asset.serialize_properties(props)])
    mask, fattrs = _float_word_mask(asset)
    for f in range(5):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawn, seed = [1500 if f == 0 else 20], [int(pcg_hash(np.array([f], dtype=np.uint32))[0])]
        ref.set_spawns(spawn, seed)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawn, seed)
        got = emu.pull()
        np.testing.assert_array_equal(got["metadata"], ref.metadata_rows())
        np.testing.assert_array_equal(got["indirect"], ref.indirect)
        np.testing.assert_array_equal(got["particles"][:, ~mask], ref.particles[:, ~mask])
        assert_float_attributes_close(got["particles"], ref.particles, fattrs, 1e-5, f"frame {f}")
        # per-step bound: restart the next step from identical state
        aos = np.ascontiguousarray(ref.particles)
        emu.lib.emu_aos_to_planes(C.byref(emu.b), aos.ctypes.data, 0, emu.rows, emu.stride)


def test_whole_frames_with_real_bookkeeping_and_ribbon_sort(orc):
    """Every kernel of hnb_simulate under emulation: hnb_init, k_bookkeeping (fused indirect + prefix sums + tile prefix),
    hnb_update, the second prefix-sum pass and both ribbon-sort kernels — a ribbon effect whose alive count crosses the
    2048-key boundary between the shared-memory sort and the cooperative radix sort."""
    from tests import static_emu
    from tests.test_gpu_ribbons import _assert_sorted, _ribbon_asset
    asset = _ribbon_asset(3000)
    fields, size, _ = asset.particle_layout()
    ref = RefWorld(3000, size // 4, [Instance(0, 3000, alive=0, seed=3)], dt=1 / 30)
    ref.set_sort_keys(fields)
    eo = EffectOracle(asset)
    emu = EmuWorld(ref, asset.generate(), chunks=1, update_ctas=2, static_lib=static_emu.build())
    crossed = False
    for f in range(10):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawn, seed = [900 if f % 3 == 0 else 23], [3]
        ref.set_spawns(spawn, seed)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawn, seed)
        _assert_sorted(ref)
        _assert_same(ref, emu.pull(), f"frame {f}")
        crossed |= ref.metadata[0].alive_count > 2048
    assert crossed


def test_real_bookkeeping_kernel_in_multi_instance_frames(orc):
    """The fused bookkeeping kernel inside whole frames with spawns: deferred init accounting for eight instances."""
    from tests import static_emu
    asset = _drifting_sparks(1)
    _, size, _ = asset.particle_layout()
    caps = [300, 64, 1000, 5, 128, 700, 33, 256]
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=10 + i))
        off += c
    ref = RefWorld(off, size // 4, insts, dt=1 / 20)
    eo = EffectOracle(asset)
    emu = EmuWorld(ref, asset.generate(), chunks=1, update_ctas=2, static_lib=static_emu.build())
    rng = np.random.default_rng(1)
    for f in range(6):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawns = [int(rng.integers(0, c + 20)) if rng.random() < 0.7 else 0 for c in caps]   # some exceed the free slots
        seeds = [int(pcg_hash(np.array([f * 16 + i], dtype=np.uint32))[0]) for i in range(len(caps))]
        ref.set_spawns(spawns, seeds)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawns, seeds)
        _assert_same(ref, emu.pull(), f"frame {f}")


@pytest.mark.parametrize("seed", range(14))
def test_random_worlds_through_every_kernel(orc, seed):
    """Fuzz of the kernels' index arithmetic: random instance layouts (capacities around tile multiples, empty and
    full instances), random spawn requests (some beyond the free slots), random tile size and grid, whole frames with
    the real bookkeeping kernel — every buffer bit-exact against the oracle after every frame."""
    from tests import static_emu
    rng = np.random.default_rng(1000 + seed)
    asset = _drifting_sparks(1) if seed % 2 else _firework_trails(1)
    _, size, _ = asset.particle_layout()
    n_inst = int(rng.integers(1, 7))
    caps = [int(rng.choice([1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 400, 511, 512, 513, 900])) for _ in range(n_inst)]
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=seed * 100 + i))
        off += c
    dt = float(rng.choice([1 / 10, 1 / 20, 1 / 4]))
    ref = RefWorld(off, size // 4, insts, dt=dt)
    eo = EffectOracle(asset)
    chunks, ctas = int(rng.choice([1, 2, 3, 4])), int(rng.integers(1, 4))
    emu = EmuWorld(ref, asset.generate(), chunks=chunks, update_ctas=ctas, static_lib=static_emu.build())
    for f in range(5):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawns = [int(rng.integers(0, c + 40)) if rng.random() < 0.6 else 0 for c in caps]
        seeds = [int(pcg_hash(np.array([seed * 64 + f * 8 + i], dtype=np.uint32))[0]) for i in range(n_inst)]
        ref.set_spawns(spawns, seeds)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawns, seeds)
        _assert_same(ref, emu.pull(), f"seed {seed} (caps {caps}, chunks {chunks}, ctas {ctas}) frame {f}")


def test_emulated_parent_child_spawn_events(orc):
    """GPU spawn events under emulation (tests/kernel_emu.py::EmuScene): the parent's update kernel appends events with
    atomics, the bookkeeping kernel accounts the event-driven child init and clears the counts, the child's init kernel
    reads the parent's records. Same scenario and same comparison rules as tests/test_gpu_events.py (event buffers as
    multisets — their order is scheduling-dependent here too —, everything else exact)."""
    from collections import Counter
    from tests import static_emu
    from tests.kernel_emu import EmuScene
    from tests.test_gpu_events import EVENT_CAP, _assets, _oracle_append_events, _oracle_child_init
    parent, child = _assets()
    p_fx, c_fx = parent.generate(num_event_bindings=1), child.generate(parent=parent)
    dt = 1.0 / 30.0
    pw = RefWorld(512, p_fx.particle_stride // 4, [Instance(0, 512, alive=0, seed=11)], dt=dt)
    cw = RefWorld(2048, c_fx.particle_stride // 4, [Instance(0, 2048, alive=0, seed=22)], dt=dt)
    po, co = EffectOracle(parent), EffectOracle(child)
    scene = EmuScene([dict(ref=pw, lowered=p_fx, emit=[0], base_child_row=0),
                      dict(ref=cw, lowered=c_fx, parent=0, consume=0, child_row=0)], [EVENT_CAP], static_emu.build())
    events, event_count, all_emitted = np.zeros(EVENT_CAP, dtype=np.uint32), 0, []
    spawn_sched = [40, 0, 25, 0, 0, 60, 0, 0, 10, 0, 0, 0, 30, 0]
    total_children = 0
    for f, spawn in enumerate(spawn_sched):
        seed_p = int(pcg_hash(np.array([100 + f], dtype=np.uint32))[0])
        seed_c = int(pcg_hash(np.array([900 + f], dtype=np.uint32))[0])
        # what the previous frame's update left in the buffer
        assert int(scene.child_infos[0, 1]) == event_count
        n_valid = min(event_count, EVENT_CAP)
        got = scene.events[0].copy()
        if event_count <= EVENT_CAP:
            assert sorted(got[:n_valid].tolist()) == sorted(events[:n_valid].tolist())
        else:
            emitted, kept = Counter(all_emitted), Counter(got.tolist())
            assert all(kept[p] <= emitted[p] for p in kept)
        events[:n_valid] = got[:n_valid]
        # ----- oracle frame (same order of passes as hnb_simulate: parent init, child init, bookkeeping, updates)
        t = np.float32(f * dt)
        pw.sim.time = cw.sim.time = t
        pw.set_spawns([spawn], [seed_p])
        cw.set_spawns([0], [seed_c])
        po.init_pass(pw)
        total_children += _oracle_child_init(child, co, cw, po, pw, events, n_valid, seed_c)
        event_count = 0
        for w in (pw, cw):
            w.oracle_indirect(orc)
            w.oracle_prefix_sum(orc)
        po.update_pass(pw)
        co.update_pass(cw)
        for channel, counts in po.last_emitted:
            event_count = _oracle_append_events(pw, counts, events, event_count)
            rows_read = pw.indirect[:pw.metadata[0].max_update, 1 - pw.metadata[0].indirect_write_index]
            all_emitted = np.repeat(rows_read, counts[:len(rows_read)]).tolist()
        # ----- emulated frame
        scene.frame_step(pw.sim, [spawn, 0], [seed_p, seed_c])
        for b, world in enumerate((pw, cw)):
            got_w = scene.pull(b)
            want_md = world.metadata_rows()[0].copy()
            want_md[5] = b
            for fld in (7, 8, 9, 10):
                want_md[fld] = got_w["metadata"][fld]
            np.testing.assert_array_equal(got_w["metadata"], want_md, err_msg=f"frame {f} member {b}: metadata")
            assert got_w["instance_count"] == world.draw[1]
            np.testing.assert_array_equal(got_w["indirect"], world.indirect, err_msg=f"frame {f} member {b}: lists")
            np.testing.assert_array_equal(got_w["particles"], world.particles, err_msg=f"frame {f} member {b}: particles")
    assert total_children > 100


def test_emulated_ordered_spawn_events(orc):
    """HNB_EFFECT_ORDERED_EVENTS under emulation: one parent, two channels (Always with a random count, OnDie x4), two
    children, buffers that overflow. With ordered append the event buffers — and therefore both children — must equal
    the oracle's canonical (serial thread order) result EXACTLY, frame after frame, overflow included."""
    from tests import static_emu
    from tests.kernel_emu import EmuScene
    from tests.test_gpu_events import EVENT_CAP, _oracle_append_events, _oracle_child_init
    wp = G.ExprWriter()
    parent = (G.EffectAsset(1024, wp.module, name="emitter")
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
    dt = 1.0 / 30.0
    pw = RefWorld(1024, p_fx.particle_stride // 4, [Instance(0, 1024, alive=0, seed=1)], dt=dt)
    cw = [RefWorld(4096, c_fx[0].particle_stride // 4, [Instance(0, 4096, alive=0, seed=2 + k)], dt=dt) for k in (0, 1)]
    po, co = EffectOracle(parent), [EffectOracle(c) for c in children]
    # members in batch order: children first (EffectSorter), then the parent; child infos / buffers 0, 1 = channels 0, 1
    scene = EmuScene([dict(ref=cw[0], lowered=c_fx[0], parent=2, consume=0, child_row=0),
                      dict(ref=cw[1], lowered=c_fx[1], parent=2, consume=1, child_row=1),
                      dict(ref=pw, lowered=p_fx, emit=[0, 1], base_child_row=0, ordered=True)], [EVENT_CAP, EVENT_CAP], static_emu.build())
    events = [np.zeros(EVENT_CAP, dtype=np.uint32) for _ in (0, 1)]
    event_count, spawned, overflowed = [0, 0], [0, 0], False
    spawn_sched = [700, 0, 0, 150, 0, 0, 0, 800, 0, 0, 0, 0, 100, 0]
    for f, spawn in enumerate(spawn_sched):
        seed_p = int(pcg_hash(np.array([5000 + f], dtype=np.uint32))[0])
        seed_c = [int(pcg_hash(np.array([6000 + 10 * f + k], dtype=np.uint32))[0]) for k in (0, 1)]
        # the buffers as the previous frame's ordered append left them: EXACTLY the canonical sequence
        for k in (0, 1):
            assert int(scene.child_infos[k, 1]) == event_count[k], f"frame {f} channel {k}: event count"
            nv = min(event_count[k], EVENT_CAP)
            overflowed |= event_count[k] > EVENT_CAP
            np.testing.assert_array_equal(scene.events[k][:nv], events[k][:nv], err_msg=f"frame {f} channel {k}: event order")
        n_valid = [min(event_count[k], EVENT_CAP) for k in (0, 1)]
        t = np.float32(f * dt)
        pw.sim.time = t
        for k in (0, 1):
            cw[k].sim.time = t
            cw[k].set_spawns([0], [seed_c[k]])
            spawned[k] += _oracle_child_init(children[k], co[k], cw[k], po, pw, events[k], n_valid[k], seed_c[k])
        pw.set_spawns([spawn], [seed_p])
        po.init_pass(pw)
        event_count = [0, 0]
        for w in (cw[0], cw[1], pw):
            w.oracle_indirect(orc)
            w.oracle_prefix_sum(orc)
        for k in (0, 1):
            co[k].update_pass(cw[k])
        po.update_pass(pw)
        for channel, counts in po.last_emitted:
            event_count[channel] = _oracle_append_events(pw, counts, events[channel], event_count[channel])
        scene.frame_step(pw.sim, [0, 0, spawn], [seed_c[0], seed_c[1], seed_p])
        for b, world in enumerate((cw[0], cw[1], pw)):
            got = scene.pull(b)
            want_md = world.metadata_rows()[0].copy()
            want_md[5] = b
            for fld in (7, 8, 9, 10):
                want_md[fld] = got["metadata"][fld]
            np.testing.assert_array_equal(got["metadata"], want_md, err_msg=f"frame {f} member {b}: metadata")
            np.testing.assert_array_equal(got["indirect"], world.indirect, err_msg=f"frame {f} member {b}: lists")
            np.testing.assert_array_equal(got["particles"], world.particles, err_msg=f"frame {f} member {b}: particles")
    assert spawned[0] > 100 and spawned[1] > 100 and overflowed


@pytest.mark.parametrize("extra", [0, 1, 2])
def test_wide_records_and_plane_tails(orc, extra):
    """Record widths that change the kernel's shape: with many attributes the tile K drops from 4 (C5) over 2 (48-byte
    trails) to 1 row per lane. (Every effect has POSITION, a vec3, so records are multiples of 16 bytes: the 8- and
    4-byte tail planes only exist for raw slabs, tests/test_gpu_misc.py::test_aos_soa_roundtrip_odd_strides.)"""
    w = G.ExprWriter()
    asset = (G.EffectAsset(700, w.module, name=f"wide{extra}")
             .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
             .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
             .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.15).uniform(w.lit(0.5))))
             .init(G.SetAttributeModifier(A.F32X4_0, w.rand(G.VEC4)))
             .init(G.SetAttributeModifier(A.HDR_COLOR, w.rand(G.VEC4) * w.lit(3.)))
             .update(G.SetAttributeModifier(A.F32X4_1, w.attr(A.F32X4_0) * w.attr(A.HDR_COLOR) + w.attr(A.F32X4_1)))
             .update(G.SetAttributeModifier(A.F32X3_0, w.attr(A.VELOCITY).cross(w.attr(A.POSITION))))
             .update(G.AccelModifier(w.lit(G.Vec3(0., -3., 0.)))))
    if extra >= 1:
        asset = asset.update(G.SetAttributeModifier(A.SIZE2, w.attr(A.SIZE2) + w.lit(G.Vec2(0.5, 0.25))))          # + an 8-byte attribute
    if extra >= 2:
        asset = (asset.update(G.SetAttributeModifier(A.F32X3_1, w.attr(A.F32X3_1) + w.attr(A.VELOCITY)))
                 .update(G.SetAttributeModifier(A.AXIS_X, w.attr(A.VELOCITY).normalize()))
                 .update(G.SetAttributeModifier(A.U32_0, w.attr(A.U32_0) + w.lit(G.U32(3)))))
    fx = asset.generate()
    _, size, _ = asset.particle_layout()
    ref = RefWorld(700, size // 4, [Instance(0, 700, alive=0, seed=5 + extra)], dt=1 / 10)
    eo = EffectOracle(asset)
    emu = EmuWorld(ref, fx, chunks=1, update_ctas=2)
    for f in range(5):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawn, seed = [500 if f == 0 else 60], [int(pcg_hash(np.array([f + 50], dtype=np.uint32))[0])]
        ref.set_spawns(spawn, seed)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawn, seed)
        _assert_same(ref, emu.pull(), f"stride {size}, frame {f}")
    print(f"stride {size} bytes, tile K {emu.lib.emu_tile_k()}")



def test_lookback_across_windows_stays_exact(orc):
    """An instance of ~70 tiles of 128 rows on 3 CTAs: a tile's look-back may have to sum more than one 32-tile window of
    predecessors before it meets a PREFIX. Results must match the oracle exactly."""
    rng = np.random.default_rng(21)
    ref = _c5_world(rng, [Instance(0, 9000, alive=8800, seed=42)])   # ~70 tiles of 128 rows: several look-back windows
    emu = EmuWorld(ref, recipes.c5_lowered(), chunks=1, update_ctas=3)
    k = (C.c_float * 4)(0.0, -9.8, 0.0, 0.5)
    for step in range(3):
        ref.oracle_frame(orc, orc.orc_body_update_c5(), k)
        emu.frame_step(orc, ref.sim, [0], [42])
        _assert_same(ref, emu.pull(), f"step {step}")


@pytest.mark.parametrize("ordered", [False, True])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_event_scenes(orc, ordered, seed):
    """Randomised parent / two-children scenes (emission probability, events per death, lifetimes, spawn schedule,
    tile size, grid). Default mode: event buffers as multisets (sub-multisets on overflow), the oracle adopts the
    buffer's order; ordered mode: exact buffers. Everything else exact in both."""
    from collections import Counter
    from tests import static_emu
    from tests.kernel_emu import EmuScene
    from tests.test_gpu_events import EVENT_CAP, _oracle_append_events, _oracle_child_init
    rng = np.random.default_rng(700 + seed)
    p_cap, c_cap = int(rng.choice([300, 1024, 1500])), 4096
    wp = G.ExprWriter()
    parent = (G.EffectAsset(p_cap, wp.module, name="emitter")
              .init(G.SetAttributeModifier(A.POSITION, wp.rand(G.VEC3) * wp.lit(2.) - wp.lit(1.)))
              .init(G.SetAttributeModifier(A.VELOCITY, wp.rand(G.VEC3) - wp.lit(0.5)))
              .init(G.SetAttributeModifier(A.AGE, wp.lit(0.)))
              .init(G.SetAttributeModifier(A.LIFETIME, wp.lit(float(rng.choice([0.05, 0.1]))).uniform(wp.lit(float(rng.choice([0.3, 0.6]))))))
              .update(G.EmitSpawnEventModifier(G.ALWAYS, (wp.rand(G.FLOAT) * wp.lit(float(rng.choice([1.0625, 1.25, 1.5])))).cast(G.UINT), 0))
              .update(G.EmitSpawnEventModifier(G.ON_DIE, wp.lit(G.U32(int(rng.integers(1, 6)))), 1)))
    children = []
    for tag in (0, 1):
        wc = G.ExprWriter()
        children.append(G.EffectAsset(c_cap, wc.module, name=f"child{tag}")
                        .init(G.InheritAttributeModifier(A.POSITION))
                        .init(G.SetAttributeModifier(A.VELOCITY, wc.parent_attr(A.VELOCITY) * wc.lit(0.5 + tag) + (wc.rand(G.VEC3) - wc.lit(0.5))))
                        .init(G.SetAttributeModifier(A.AGE, wc.lit(0.)))
                        .init(G.SetAttributeModifier(A.LIFETIME, wc.lit(0.15 + 0.1 * tag)))
                        .init(G.SetAttributeModifier(A.U32_0, wc.parent_attr(A.ID))))
    p_fx = parent.generate(num_event_bindings=2, ordered_events=ordered)
    c_fx = [c.generate(parent=parent) for c in children]
    dt = 1.0 / 30.0
    pw = RefWorld(p_cap, p_fx.particle_stride // 4, [Instance(0, p_cap, alive=0, seed=1)], dt=dt)
    cw = [RefWorld(c_cap, c_fx[0].particle_stride // 4, [Instance(0, c_cap, alive=0, seed=2 + k)], dt=dt) for k in (0, 1)]
    po, co = EffectOracle(parent), [EffectOracle(c) for c in children]
    scene = EmuScene([dict(ref=cw[0], lowered=c_fx[0], parent=2, consume=0, child_row=0),
                      dict(ref=cw[1], lowered=c_fx[1], parent=2, consume=1, child_row=1),
                      dict(ref=pw, lowered=p_fx, emit=[0, 1], base_child_row=0, ordered=ordered)], [EVENT_CAP, EVENT_CAP], static_emu.build(),
                     chunks=int(rng.choice([1, 2])), update_ctas=int(rng.integers(1, 4)))
    events = [np.zeros(EVENT_CAP, dtype=np.uint32) for _ in (0, 1)]
    event_count, all_emitted = [0, 0], [[], []]
    for f in range(10):
        spawn = int(rng.integers(0, p_cap)) if rng.random() < 0.4 else 0
        seed_p = int(pcg_hash(np.array([seed * 1000 + f], dtype=np.uint32))[0])
        seed_c = [int(pcg_hash(np.array([seed * 1000 + 500 + 10 * f + k], dtype=np.uint32))[0]) for k in (0, 1)]
        n_valid = []
        for k in (0, 1):
            assert int(scene.child_infos[k, 1]) == event_count[k]
            nv = min(event_count[k], EVENT_CAP)
            got = scene.events[k].copy()
            if ordered:
                np.testing.assert_array_equal(got[:nv], events[k][:nv], err_msg=f"frame {f} channel {k}: event order")
            elif event_count[k] <= EVENT_CAP:
                assert sorted(got[:nv].tolist()) == sorted(events[k][:nv].tolist())
            else:
                emitted, kept = Counter(all_emitted[k]), Counter(got.tolist())
                assert all(kept[p] <= emitted[p] for p in kept)
            events[k][:nv] = got[:nv]
            n_valid.append(nv)
        t = np.float32(f * dt)
        pw.sim.time = t
        for k in (0, 1):
            cw[k].sim.time = t
            cw[k].set_spawns([0], [seed_c[k]])
            _oracle_child_init(children[k], co[k], cw[k], po, pw, events[k], n_valid[k], seed_c[k])
        pw.set_spawns([spawn], [seed_p])
        po.init_pass(pw)
        event_count = [0, 0]
        for w in (cw[0], cw[1], pw):
            w.oracle_indirect(orc)
            w.oracle_prefix_sum(orc)
        for k in (0, 1):
            co[k].update_pass(cw[k])
        po.update_pass(pw)
        for channel, counts in po.last_emitted:
            event_count[channel] = _oracle_append_events(pw, counts, events[channel], event_count[channel])
            rows_read = pw.indirect[:pw.metadata[0].max_update, 1 - pw.metadata[0].indirect_write_index]
            all_emitted[channel] = np.repeat(rows_read, counts[:len(rows_read)]).tolist()
        scene.frame_step(pw.sim, [0, 0, spawn], [seed_c[0], seed_c[1], seed_p])
        for b, world in enumerate((cw[0], cw[1], pw)):
            got = scene.pull(b)
            want_md = world.metadata_rows()[0].copy()
            want_md[5] = b
            for fld in (7, 8, 9, 10):
                want_md[fld] = got["metadata"][fld]
            np.testing.assert_array_equal(got["metadata"], want_md, err_msg=f"frame {f} member {b}: metadata")
            np.testing.assert_array_equal(got["indirect"], world.indirect, err_msg=f"frame {f} member {b}: lists")
            np.testing.assert_array_equal(got["particles"], world.particles, err_msg=f"frame {f} member {b}: particles")


@pytest.mark.parametrize("name", ["c5", "trails", "ribbons", "wide"])
def test_sector_plane_layout(orc, name):
    """HNB_SLAB_SECTOR_PLANES / HNB_EFFECT_SECTOR_PLANES: pairs of 16-byte record pieces in 32-byte-wide columns (one
    DRAM sector per gathered pair). Same results as the default layout, through init, update and the ribbon sort."""
    from tests import static_emu
    from tests.test_gpu_ribbons import _ribbon_asset
    if name == "c5":
        asset = recipes.c5_asset(2000)
    elif name == "trails":
        asset = _firework_trails(2000)          # 48 bytes: one sector column + one 16-byte column
    elif name == "ribbons":
        asset = _ribbon_asset(2000)
    else:
        w = G.ExprWriter()
        asset = (G.EffectAsset(2000, w.module, name="wide_sector")
                 .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3)))
                 .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) - w.lit(0.5)))
                 .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
                 .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.2).uniform(w.lit(0.6))))
                 .init(G.SetAttributeModifier(A.F32X4_0, w.rand(G.VEC4)))
                 .init(G.SetAttributeModifier(A.HDR_COLOR, w.rand(G.VEC4)))
                 .update(G.SetAttributeModifier(A.F32X4_1, w.attr(A.F32X4_0) + w.attr(A.HDR_COLOR) * w.attr(A.F32X4_1)))
                 .update(G.SetAttributeModifier(A.F32X3_0, w.attr(A.VELOCITY).cross(w.attr(A.POSITION)))))
    fields, size, _ = asset.particle_layout()
    fx = asset.generate(sector_planes=True)
    ref = RefWorld(2000, size // 4, [Instance(0, 2000, alive=0, seed=4)], dt=1 / 10)
    if name == "ribbons":
        ref.set_sort_keys(fields)
    eo = EffectOracle(asset)
    emu = EmuWorld(ref, fx, chunks=1, update_ctas=2, static_lib=static_emu.build())
    assert emu.sector
    for f in range(6):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawn, seed = [900 if f % 3 == 0 else 40], [int(pcg_hash(np.array([f + 300], dtype=np.uint32))[0])]
        ref.set_spawns(spawn, seed)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawn, seed)
        _assert_same(ref, emu.pull(), f"{name} (stride {size}) frame {f}")


def test_kernels_with_matrix_values(orc):
    """Matrix literals and properties (matCxR<f32>; a 96-byte Properties record holding a mat2x2, a vec4 and a mat4x4)
    through the real hnb_init / hnb_update: two instances with different property records. Products only multiply
    and add in a fixed order: bit-exact against the interpreter."""
    from tests.test_host_exec_cpu import _MATRIX_PROPS, _matrix_asset
    asset = _matrix_asset(1024)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(2048, size // 4, [Instance(0, 1024, alive=0, seed=21), Instance(1024, 1024, alive=0, seed=22)], dt=1 / 20)
    props = [_MATRIX_PROPS, {}]
    for i in range(2):
        ref.metadata[i].properties_array_index = i
    eo = EffectOracle(asset, {0: props[0], 1: props[1]})
    emu = EmuWorld(ref, asset.generate(), chunks=1, update_ctas=2, property_blobs=[asset.serialize_properties(p) for p in props])
    for f in range(5):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawn = [600 if f == 0 else 30, 250 if f % 2 == 0 else 0]
        seed = [int(x) for x in pcg_hash(np.array([2 * f, 2 * f + 1], dtype=np.uint32))]
        ref.set_spawns(spawn, seed)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawn, seed)
        got = emu.pull()
        np.testing.assert_array_equal(got["metadata"], ref.metadata_rows())
        np.testing.assert_array_equal(got["indirect"], ref.indirect)
        np.testing.assert_array_equal(got["particles"], ref.particles, err_msg=f"frame {f}")
    assert ref.metadata[0].alive_count > 300 and ref.metadata[1].alive_count > 100


def test_c2_firework_at_its_baseline_size(orc):
    """BASELINE.json configs[1] ("firework.rs effect, 32768 capacity") at its quoted size: 50 frames of bursts into recycled
    slots through the emulated init / bookkeeping / update kernels with the 4-chunk tiles large slabs get. Zero tolerance."""
    from tests import static_emu
    asset = _firework_trails(32768)
    _, size, _ = asset.particle_layout()
    ref = RefWorld(32768, size // 4, [Instance(0, 32768, alive=0)], dt=1 / 20)
    eo = EffectOracle(asset)
    emu = EmuWorld(ref, asset.generate(), chunks=4, update_ctas=3, static_lib=static_emu.build())
    for f in range(50):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawn, seed = [9000 if f % 20 == 0 else 150], [int(pcg_hash(np.array([0x4321 + f], dtype=np.uint32))[0])]
        ref.set_spawns(spawn, seed)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawn, seed)
        if f % 5 == 0 or f == 49:
            _assert_same(ref, emu.pull(), f"frame {f}")
    assert ref.metadata[0].particle_counter == 34050 and ref.metadata[0].alive_count == 11768


def test_c3_force_field_at_its_baseline_size(orc):
    """BASELINE.json configs[2] ("force_field.rs: 1M particles") at its quoted size through the emulated kernels (a burst of
    1 Mi - 4096 spawns run as waves of init CTAs, then 4-chunk update tiles over the whole slab): integer structures
    exact, fp32 attributes within 1e-5 of their magnitude per step (host libm vs numpy)."""
    from tests import static_emu
    from tests.helpers import assert_float_attributes_close
    from tests.test_gpu_effects import _float_word_mask, _force_field
    n = 1 << 20
    asset = _force_field(n)
    _, size, _ = asset.particle_layout()
    props = {"attraction_accel": 18.0, "repulsor_position": G.Vec3(0.25, 0.5, 0.1)}
    ref = RefWorld(n, size // 4, [Instance(0, n, alive=0, seed=77)])
    ref.metadata[0].properties_array_index = 0
    eo = EffectOracle(asset, {0: props})
    emu = EmuWorld(ref, asset.generate(), chunks=4, update_ctas=3, static_lib=static_emu.build(), property_blobs=[asset.serialize_properties(props)])
    mask, fattrs = _float_word_mask(asset)
    for f in range(2):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        spawn, seed = [n - 4096 if f == 0 else 500], [int(pcg_hash(np.array([f], dtype=np.uint32))[0])]
        ref.set_spawns(spawn, seed)
        eo.frame(ref, orc)
        emu.frame_step(orc, ref.sim, spawn, seed)
        got = emu.pull()
        np.testing.assert_array_equal(got["metadata"], ref.metadata_rows())
        np.testing.assert_array_equal(got["indirect"], ref.indirect)
        np.testing.assert_array_equal(got["particles"][:, ~mask], ref.particles[:, ~mask])
        assert_float_attributes_close(got["particles"], ref.particles, fattrs, 1e-5, f"frame {f}")
        aos = np.ascontiguousarray(ref.particles)
        emu.lib.emu_aos_to_planes(C.byref(emu.b), aos.ctypes.data, 0, emu.rows, emu.stride)
    assert ref.metadata[0].alive_count == n - 4096 + 500


def test_tile_word_rule():
    """hnb_tile_count as restated by tile_count: ceil(rows / S) tiles, whatever flags the word carries."""
    for rows in (0, 1, 127, 128, 129, 511, 512, 513, 4700, 65536, 1 << 20):
        assert int(tile_count(rows, 512)) == (rows + 511) // 512
        assert int(tile_count(rows, 512 | 0x80000000)) == (rows + 511) // 512
