"""Batch slots that sit out, and batch slots that change hands, on the device, against the oracle.

A batch slot (batch_info_index) keeps its array of look-back tile states from frame to frame. Slot-order state words keep
only 6 bits of epoch, so a word written 64 frames earlier passes for current unless the host zeroes the array
(tile_state_rule.h): that is the case when a batch sits out for 63 frames (or 127, ...) and comes back, or when a slot
serves an instance with fewer tiles in between. Default-order words carry 30 bits of epoch and relaxed order runs no
look-back, but their frame-to-frame reuse is exercised here too.

One context holds several instances (metadata, draw-args and spawner rows of their own) in one or two slabs; every frame
uploads the spawner and batch tables of the batches that run, as a host that pauses an effect does, and the oracle runs
exactly those batches. After every frame every slab is compared bit for bit (instances that sat out must be unchanged),
as are the metadata and draw-args rows of every instance and the frame's prefix sums, batch infos, dispatch args and
render indices; relaxed order compares the lists as sets. The tile-state clears the context made are checked after every
frame against the rule, restated. Whether a stale word would actually be read depends on timing, so the scenarios give
it chances: many 128-row tiles per instance, alternating full and empty 128-row spans (an empty bitmap word skips the
record loads, so a successor often finishes its first pass before its predecessor), and populations that keep changing.
The CPU model (tests/test_tile_state_epochs_cpu.py) is the deterministic guard.
"""
import ctypes as C

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N, graph as G, recipes
from oracle import c_oracle as O
from oracle.hanabi_oracle import EffectOracle
from tests.helpers import RefWorld
from tests.test_gpu_update_c5 import ACCEL_DRAG

pytestmark = pytest.mark.gpu
A = G.Attribute
EPOCH_MASK = 0x3FFFFFFF
ORDERS = ["default", "slot", "relaxed"]
# relaxed order hands out recycled slots in a scheduling-dependent order, so the spawning effect runs in the other two
ORDER_KIND = [(o, "c5") for o in ORDERS] + [("default", "sparks"), ("slot", "sparks")]


def _sparks(capacity):
    w = G.ExprWriter()
    return (G.EffectAsset(capacity, w.module, name="sparks_batch_slots")
            .init(G.SetAttributeModifier(A.POSITION, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
            .init(G.SetAttributeModifier(A.VELOCITY, w.rand(G.VEC3) * w.lit(2.) - w.lit(1.)))
            .init(G.SetAttributeModifier(A.AGE, w.lit(0.)))
            .init(G.SetAttributeModifier(A.LIFETIME, w.lit(0.05).uniform(w.lit(0.4))))
            .update(G.AccelModifier(w.lit(G.Vec3(0., -9.8, 0.))))
            .update(G.LinearDragModifier(w.lit(0.5))))


class Scene:
    """One context, its slabs and instances, driven frame by frame with an arbitrary list of batches."""

    def __init__(self, ctx, orc):
        self.ctx, self.orc = ctx, orc
        self.slabs, self.insts, self.effects = {}, [], {}
        self.dt = 1.0 / 60.0
        self.frames = 0
        self.expected_clears = 0
        self.slot_record = {}      # batch slot -> [signature, first epoch] (tile_state_rule.h restated)
        self.relaxed_slabs = set()  # slabs a relaxed-order batch has written: their lists are compared as sets from then on
        self.body = orc.orc_body_update_c5()

    # ---- setup --------------------------------------------------------------------------------------------------------
    def slab(self, name, rows, stride_words):
        particles = np.zeros((rows, stride_words), dtype=np.uint32)
        indirect = np.zeros((rows, 3), dtype=np.uint32)
        indirect[:, 2] = np.arange(rows, dtype=np.uint32)
        self.slabs[name] = dict(rows=rows, stride_words=stride_words, particles=particles, indirect=indirect, handle=None, slot_order=False)

    def effect(self, name, kind, order):
        """kind "c5": C5 (deaths only, C oracle); "sparks": spawning, numpy oracle. One handle per name: two names of the same
        code are two effects to the context."""
        if kind == "c5":
            lowered = recipes.c5_lowered(relaxed_order=order == "relaxed", slot_order=order == "slot")
            eo = None
        else:
            asset = _sparks(4096)
            lowered = asset.generate(relaxed_order=order == "relaxed", slot_order=order == "slot")
            eo = EffectOracle(asset)
        self.effects[name] = dict(kind=kind, order=order, handle=self.ctx.effect_compile(lowered), oracle=eo, stride=lowered.particle_stride)

    def instance(self, slab, offset, capacity, rng, alive_rows=None, life=(0.02, 0.6), seed=0):
        """`alive_rows`: rows of the instance alive at the start (default none), ascending; C5 records with random motion."""
        s = self.slabs[slab]
        alive_rows = np.asarray(alive_rows if alive_rows is not None else [], dtype=np.int64)
        n = len(alive_rows)
        dead_rows = np.setdiff1d(np.arange(capacity), alive_rows)
        s["indirect"][offset:offset + n, 0] = alive_rows
        s["indirect"][offset:offset + n, 1] = alive_rows
        s["indirect"][offset + n:offset + capacity, 2] = offset + dead_rows
        if n:
            p = np.zeros((n, 8), dtype=np.float32)
            p[:, 0:3] = rng.uniform(-1, 1, (n, 3))
            p[:, 4:7] = rng.uniform(-1, 1, (n, 3))
            p[:, 7] = rng.uniform(*life, n)
            s["particles"][offset + alive_rows] = p.view(np.uint32)
        row = len(self.insts)
        md = O.EffectMetadata()
        md.capacity, md.alive_count, md.max_update, md.max_spawn = capacity, n, 0, capacity - n
        md.indirect_write_index, md.indirect_render_index = 0, row
        for f in ("init_indirect_dispatch_index", "properties_array_index", "local_child_index", "global_child_index",
                  "base_child_index", "sort_key_offset", "sort_key2_offset"):
            setattr(md, f, 0xFFFFFFFF)
        md.particle_stride = s["stride_words"]
        sp = O.Spawner()
        sp.transform, sp.inverse_transform = O.identity_rows(), O.identity_rows()
        sp.seed, sp.effect_metadata_index, sp.draw_indirect_index = seed, row, row
        sp.slab_offset, sp.parent_slab_offset = offset, 0xFFFFFFFF
        self.insts.append(dict(slab=slab, offset=offset, capacity=capacity, md=md, sp=sp, draw=np.zeros(5, dtype=np.uint32)))
        return row

    def upload(self, slot_order_slabs=()):
        """Everything to the device once: metadata rows are inserted here only (an insert changes every signature)."""
        ctx = self.ctx
        for name, s in self.slabs.items():
            s["handle"] = ctx.slab_create(s["rows"], s["stride_words"] * 4)
            ctx.slab_upload_aos(s["handle"], 0, s["particles"])
            ctx.slab_upload_indirect(s["handle"], 0, s["indirect"])
        for i, inst in enumerate(self.insts):
            if inst["slab"] in slot_order_slabs:
                ctx.slab_rebuild_alive_bits(self.slabs[inst["slab"]]["handle"], inst["offset"], inst["capacity"], 0, inst["md"].alive_count)
            ctx.metadata_insert(i, N.EffectMetadata.from_buffer_copy(bytes(inst["md"])))
            ctx.draw_args_insert(i, N.DrawIndexedIndirectArgs(*[int(x) for x in inst["draw"]]))
        ctx.sync()

    # ---- one frame ------------------------------------------------------------------------------------------------------
    def frame(self, batches, spawns=None):
        """batches: [(effect name, [instance rows])], batch slot = position in the list. spawns: {instance row: count}."""
        spawns = spawns or {}
        self.frames += 1
        rows = [i for _, members in batches for i in members]
        E, B = len(rows), len(batches)
        fw = object.__new__(RefWorld)                          # the oracle's view of this frame's tables
        fw.sim = O.SimParams(self.dt, np.float32(self.frames) * np.float32(self.dt), self.dt, 0.0, self.dt, 0.0, E)
        fw.spawners, fw.metadata = (O.Spawner * max(E, 1))(), (O.EffectMetadata * max(E, 1))()
        fw.draw = np.zeros(5 * max(E, 1), dtype=np.uint32)
        fw.prefix = np.zeros(max(E, 1), dtype=np.uint32)
        fw.batches, fw.batch_infos, fw.dispatch = [], (O.BatchInfo * max(B, 1))(), np.zeros(3 * max(B, 1), dtype=np.uint32)
        dev_sp = (N.Spawner * max(E, 1))()
        cpu_prefix = []
        j = 0
        for b, (_, members) in enumerate(batches):
            fw.batches.append(list(range(j, j + len(members))))
            bi = fw.batch_infos[b]
            bi.spawner_base, bi.base_particle, bi.prefix_sum_offset, bi.prefix_sum_count = j, self.insts[members[0]]["offset"], j, len(members)
            run = 0
            for i in members:
                inst = self.insts[i]
                inst["sp"].spawn = int(spawns.get(i, 0))
                inst["sp"].seed = (1000 + 17 * self.frames + i) & 0xFFFFFFFF
                sp = O.Spawner.from_buffer_copy(bytes(inst["sp"]))
                dev_sp[j] = N.Spawner.from_buffer_copy(bytes(sp))
                sp.effect_metadata_index = sp.draw_indirect_index = j
                fw.spawners[j] = sp
                md = O.EffectMetadata.from_buffer_copy(bytes(inst["md"]))
                md.indirect_render_index = j
                fw.metadata[j] = md
                fw.draw[5 * j:5 * j + 5] = inst["draw"]
                cpu_prefix.append(run)
                fw.prefix[j] = run
                run += max(0, inst["sp"].spawn)
                j += 1
        # ---- the oracle: init -> indirect -> prefix sum -> update over exactly these batches
        def on_slab(b):
            s = self.slabs[self.insts[batches[b][1][0]]["slab"]]
            fw.particles, fw.indirect = s["particles"], s["indirect"]
            fx = self.effects[batches[b][0]]
            fw.slot_order, fw.stride_words = fx["order"] == "slot", s["stride_words"]
            return fx
        for b in range(B):
            fx = on_slab(b)
            if fx["oracle"] is not None:
                fx["oracle"].init_pass(fw, b)
        fw.oracle_indirect(self.orc)
        fw.oracle_prefix_sum(self.orc)
        for b in range(B):
            fx = on_slab(b)
            if fx["oracle"] is not None:
                fx["oracle"].update_pass(fw, b)
            else:
                fw.oracle_update(self.orc, self.body, ACCEL_DRAG, b)
        for j, i in enumerate(rows):                           # back into the instances' own rows
            inst = self.insts[i]
            md = O.EffectMetadata.from_buffer_copy(bytes(fw.metadata[j]))
            md.indirect_render_index = i
            inst["md"] = md
            sp = O.Spawner.from_buffer_copy(bytes(fw.spawners[j]))
            sp.effect_metadata_index = sp.draw_indirect_index = i
            inst["sp"] = sp
            inst["draw"] = fw.draw[5 * j:5 * j + 5].copy()
        # ---- the device: the same tables
        ctx = self.ctx
        run_epoch = (ctx.last_epoch() + 1) & EPOCH_MASK or 1
        ctx.upload_spawners_raw(dev_sp, E)
        ctx.upload_batches_raw((N.BatchInfo * max(B, 1)).from_buffer_copy(bytes(fw.batch_infos)), B, (N.u32 * max(E, 1))(*cpu_prefix), E)
        N.check(N.lib.hnb_set_sim_params(ctx._h, C.byref(N.SimParams.from_buffer_copy(bytes(fw.sim)))))
        launches = []
        for b, (name, members) in enumerate(batches):
            fx, s = self.effects[name], self.slabs[self.insts[members[0]]["slab"]]
            launches.append(N.BatchLaunch.make(fx["handle"], s["handle"], b, sum(max(0, spawns.get(i, 0)) for i in members)))
            self._expect_clear(b, fx, s, len(members), fw.batch_infos[b].spawner_base, run_epoch)
        ctx.simulate(launches)
        assert ctx.last_epoch() == run_epoch
        self.check(fw, batches, rows)

    def _expect_clear(self, b, fx, s, count, spawner_base, run_epoch):
        """tile_state_rule.h restated: a slot-order batch zeroes its states when its signature changes (its first run
        included) and 64 or more epochs after the first run since the last zeroing; a batch of another order only when
        its slot served slot order before. The tile word follows from effect, slab and count here, and the metadata
        rows are never re-inserted."""
        sig = (fx["handle"], s["handle"], count, spawner_base) if fx["order"] == "slot" else None
        rec = self.slot_record.get(b)
        if sig is None:
            if rec is not None and rec[0] is not None:
                self.expected_clears += 1
            self.slot_record[b] = [None, 0]
            return
        if rec is None or rec[0] != sig:
            self.expected_clears += 1
            self.slot_record[b] = [sig, run_epoch]
        elif run_epoch < rec[1]:
            rec[1] = run_epoch
        elif run_epoch - rec[1] >= 64:
            self.expected_clears += 1
            rec[1] = run_epoch

    # ---- the comparison ------------------------------------------------------------------------------------------------
    def check(self, fw, batches, rows):
        ctx, what = self.ctx, f"frame {self.frames}"
        ctx.sync()
        assert ctx.tile_state_clears() == self.expected_clears, f"{what}: tile-state clears"
        for i, inst in enumerate(self.insts):
            got = np.frombuffer(bytes(ctx.read_metadata(i)), dtype=np.uint32)
            np.testing.assert_array_equal(got, np.frombuffer(bytes(inst["md"]), dtype=np.uint32), err_msg=f"{what}: metadata row {i}")
            got = np.frombuffer(bytes(ctx.read_draw_args(i)), dtype=np.uint32)
            np.testing.assert_array_equal(got, inst["draw"], err_msg=f"{what}: draw args row {i}")
        E, B = len(rows), len(batches)
        if E:
            np.testing.assert_array_equal(np.array(ctx.read_prefix_sum(0, E), dtype=np.uint32), fw.prefix[:E], err_msg=f"{what}: prefix sums")
            rp = [ctx.read_spawner(j).render_pong for j in range(E)]
            assert rp == [fw.spawners[j].render_indirect_read_index for j in range(E)], f"{what}: spawner.render_pong"
        for b in range(B):
            got = np.frombuffer(bytes(ctx.read_batch_info(b)), dtype=np.uint32)
            np.testing.assert_array_equal(got, np.frombuffer(bytes(fw.batch_infos[b]), dtype=np.uint32), err_msg=f"{what}: batch info {b}")
            got = np.frombuffer(bytes(ctx.read_dispatch_args(b)), dtype=np.uint32)
            np.testing.assert_array_equal(got, fw.dispatch[3 * b:3 * b + 3], err_msg=f"{what}: dispatch args {b}")
        self.relaxed_slabs |= {self.insts[i]["slab"] for name, members in batches for i in members if self.effects[name]["order"] == "relaxed"}
        relaxed = self.relaxed_slabs
        for name, s in self.slabs.items():
            aos = ctx.slab_download_aos(s["handle"], 0, s["rows"], s["stride_words"] * 4)
            ind = ctx.slab_download_indirect(s["handle"], 0, s["rows"])
            np.testing.assert_array_equal(aos, s["particles"], err_msg=f"{what}: slab {name} particles")
            if name not in relaxed:
                np.testing.assert_array_equal(ind, s["indirect"], err_msg=f"{what}: slab {name} indirect (ping/pong/dead)")
                continue
            for inst in self.insts:                            # relaxed order: each instance's lists as sets
                if inst["slab"] != name:
                    continue
                md, base, cap = inst["md"], inst["offset"], inst["capacity"]
                n, W = md.alive_count, md.indirect_write_index
                assert sorted(ind[base:base + n, W].tolist()) == sorted(s["indirect"][base:base + n, W].tolist()), f"{what}: alive set"
                assert sorted(ind[base + n:base + cap, 2].tolist()) == sorted(s["indirect"][base + n:base + cap, 2].tolist()), f"{what}: dead set"

    def bitmap_consistent(self):
        assert self.ctx.read_debug(False)[15] == 0, "alive bitmap and counters disagree"


def _striped(capacity, rng, span=128, density=1.0):
    """Alternating full and empty `span`-row spans (the full ones at `density`)."""
    rows = np.arange(capacity)
    keep = ((rows // span) % 2 == 0) & (rng.random(capacity) < density)
    return rows[keep]


def _two_instances(ctx, orc, order, caps, rng, kind="c5"):
    """X and Y in one slab, one effect: the signature of a batch of Y (or of X) is the same whenever it runs."""
    sc = Scene(ctx, orc)
    off_y = (caps[0] + 127) // 128 * 128
    sc.slab("s", off_y + caps[1], 8)
    sc.effect("fx", kind, order)
    alive = (lambda c: _striped(c, rng, density=0.9)) if kind == "c5" else (lambda c: None)
    sc.instance("s", 0, caps[0], rng, alive(caps[0]), life=(0.02, 3.0), seed=1)
    sc.instance("s", off_y, caps[1], rng, alive(caps[1]), life=(0.02, 3.0), seed=2)
    sc.upload(slot_order_slabs=("s",) if order == "slot" else ())
    return sc


def _spawns(sc, kind, rows):
    if kind != "sparks":
        return {}
    return {i: (sc.insts[i]["capacity"] // 6 if sc.frames % 2 == 0 else sc.insts[i]["capacity"] // 11) for i in rows}


@pytest.mark.parametrize("order,kind", ORDER_KIND)
def test_sit_out(ctx, orc, order, kind):
    """X in slot 0 runs every frame; Y in slot 1 is absent for N frames, then runs for several frames."""
    rng = np.random.default_rng(7)
    sc = _two_instances(ctx, orc, order, (8192, 16384), rng, kind)
    X, Y = 0, 1
    for n in (1, 63, 64, 65, 127, 128):
        for _ in range(3):
            sc.frame([("fx", [X]), ("fx", [Y])], _spawns(sc, kind, [X, Y]))
        for _ in range(n):
            sc.frame([("fx", [X])], _spawns(sc, kind, [X]))
        for _ in range(4):
            sc.frame([("fx", [X]), ("fx", [Y])], _spawns(sc, kind, [X, Y]))
    if order == "slot":
        sc.bitmap_consistent()
        assert sc.expected_clears > 2 + 5, "Y's returns after 63 frames and more zeroed its states"
    else:
        assert sc.expected_clears == 0


@pytest.mark.parametrize("order", ORDERS)
def test_empty_frames(ctx, orc, order):
    """64 and 128 frames with no batch at all, then both batches resume."""
    rng = np.random.default_rng(8)
    sc = _two_instances(ctx, orc, order, (4096, 12288), rng)
    for gap in (64, 128, 63):
        for _ in range(3):
            sc.frame([("fx", [0]), ("fx", [1])])
        for _ in range(gap):
            sc.frame([])
        for _ in range(3):
            sc.frame([("fx", [0]), ("fx", [1])])
    if order == "slot":
        sc.bitmap_consistent()
        assert sc.expected_clears > 2, "the returns zeroed the states"
    else:
        assert sc.expected_clears == 0


@pytest.mark.parametrize("frames_y", [63, 64])
@pytest.mark.parametrize("order,kind", ORDER_KIND)
def test_hand_over_same_signature(ctx, orc, order, kind, frames_y):
    """Slot 0 serves X (8192 slots), then Y (4096 slots, same effect and slab: the same signature) for 63 / 64 frames, then
    X again: X's upper tiles find the words they wrote before the hand-over."""
    rng = np.random.default_rng(9)
    sc = _two_instances(ctx, orc, order, (8192, 4096), rng, kind)
    for rounds in range(2):
        for _ in range(2):
            sc.frame([("fx", [0])], _spawns(sc, kind, [0]))
        for _ in range(frames_y):
            sc.frame([("fx", [1])], _spawns(sc, kind, [1]))
        for _ in range(4):
            sc.frame([("fx", [0])], _spawns(sc, kind, [0]))
    if order == "slot":
        sc.bitmap_consistent()
        assert sc.expected_clears >= 2, "the slot's states were zeroed before X returned"
    else:
        assert sc.expected_clears == 0


@pytest.mark.parametrize("order", ["default", "slot"])
def test_hand_over_between_effects_and_slabs(ctx, orc, order):
    """Slot 0 changes effect (two handles of the same code) and slab from frame to frame: the signature part of the rule."""
    rng = np.random.default_rng(10)
    sc = Scene(ctx, orc)
    sc.slab("a", 8192 + 4096, 8)
    sc.slab("b", 6144, 8)
    sc.effect("e1", "c5", order)
    sc.effect("e2", "c5", order)
    sc.instance("a", 0, 8192, rng, _striped(8192, rng, density=0.9), life=(0.02, 2.0), seed=1)
    sc.instance("a", 8192, 4096, rng, _striped(4096, rng, density=0.9), life=(0.02, 2.0), seed=2)
    sc.instance("b", 0, 6144, rng, _striped(6144, rng, density=0.9), life=(0.02, 2.0), seed=3)
    sc.upload(slot_order_slabs=("a", "b") if order == "slot" else ())
    plan = [("e1", [0])] * 3 + [("e2", [1])] * 3 + [("e1", [2])] * 3 + [("e2", [0])] * 2 + [("e1", [1])] + [("e2", [2])] * 2
    for _ in range(3):
        for name, members in plan:
            sc.frame([(name, members)])
    if order == "slot":
        sc.bitmap_consistent()
        assert sc.expected_clears > 10
    else:
        assert sc.expected_clears == 0


@pytest.mark.parametrize("order", ["default", "slot"])
def test_sit_out_across_the_epoch_wrap(native, orc, monkeypatch, order):
    """Epochs start just below 2^30: Y sits out for 64 frames across the 30-bit wrap, then both run on."""
    monkeypatch.setenv("HNB_EPOCH_START", str(EPOCH_MASK - 30))
    c = native.Context(0)
    try:
        rng = np.random.default_rng(11)
        sc = _two_instances(c, orc, order, (4096, 8192), rng)
        for _ in range(3):
            sc.frame([("fx", [0]), ("fx", [1])])
        for _ in range(64):
            sc.frame([("fx", [0])])
        assert c.last_epoch() < 64, "the sit-out spans the wrap"
        for _ in range(70):
            sc.frame([("fx", [0]), ("fx", [1])])
    finally:
        c.close()


def test_slot_order_refuses_a_slab_of_2_28_rows(ctx, native):
    """Slot-order state words pack each count into 28 bits: such a slab is refused before anything is enqueued. The smallest
    stride there is (position + age, 16 bytes) keeps the slab at about 7 GiB with its index columns."""
    w = G.ExprWriter()
    asset = (G.EffectAsset(1024, w.module, name="tiny_slot_order")
             .init(G.SetAttributeModifier(A.POSITION, w.lit(G.Vec3(0., 0., 0.))))
             .init(G.SetAttributeModifier(A.AGE, w.lit(0.))))
    lowered = asset.generate(slot_order=True)
    rows = 1 << 28
    need = rows * (lowered.particle_stride + 12)
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < need + (1 << 30) or free < 8 << 30:
        pytest.skip(f"needs {(need >> 30) + 1} GiB of free device memory, {free >> 30} GiB free")
    fx = ctx.effect_compile(lowered)
    slab = ctx.slab_create(rows, lowered.particle_stride)
    md = N.EffectMetadata()
    md.capacity, md.max_spawn, md.particle_stride = rows, rows, lowered.particle_stride // 4
    ctx.metadata_insert(0, md)
    sp = (N.Spawner * 1)()
    sp[0].effect_metadata_index, sp[0].draw_indirect_index, sp[0].slab_offset, sp[0].parent_slab_offset = 0, 0, 0, 0xFFFFFFFF
    ctx.upload_spawners_raw(sp, 1)
    ctx.upload_batches_raw((N.BatchInfo * 1)(N.BatchInfo(0, 0, 0, 0, 0, 1)), 1, (N.u32 * 1)(0), 1)
    ctx.sync()
    epoch, clears = ctx.last_epoch(), ctx.tile_state_clears()
    with pytest.raises(N.HanabiError) as e:
        ctx.simulate([N.BatchLaunch.make(fx, slab, 0, 0)])
    assert e.value.code == N.HNB_ERR_LAYOUT and "2^28" in e.value.message
    ctx.sync()
    assert ctx.last_epoch() == epoch and ctx.tile_state_clears() == clears
    assert bytes(ctx.read_metadata(0)) == bytes(md)
    ctx.slab_destroy(slab)
