"""Shared test scaffolding: one "world" (a slab + its instances + per-frame tables) kept in the
reference's own layouts, which can be stepped by the C oracle and mirrored onto / read back from the GPU
backend through the C ABI.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Sequence

import numpy as np
import pytest

from oracle import c_oracle as O
from oracle.hanabi_oracle import pcg_hash

SUB_TILE_C5 = 128  # rows of an update sub-tile for C5 records: 32 lanes x K = 4 rows in flight per lane


@pytest.fixture(params=[1, 2, 3, 4], ids=lambda n: f"{n}sub")
def tiled_ctx(request, native, monkeypatch):
    """A fresh context on cuda:0 whose update tiles hold `tile_chunks` sub-tiles, forced with HNB_TILE_CHUNKS (None: the
    slab-size rule of tile_chunks, which picks 1 below one wave of resident warps, about 400 Ki rows for C5, so without the
    override almost every row-exact test would run 1). The results are the same at every tile size by design, so after a
    forced run the fixture reads back the tile size of the last launch of batch `tile_batch` (default 0; its effect must
    have records of at most 36 bytes, as C5's, for 128-row sub-tiles) to prove that the size under test was the one that
    ran."""
    chunks = request.param
    if chunks is None:
        monkeypatch.delenv("HNB_TILE_CHUNKS", raising=False)
    else:
        monkeypatch.setenv("HNB_TILE_CHUNKS", str(chunks))
    c = native.Context(0)
    c.tile_chunks, c.tile_batch = chunks, 0
    try:
        yield c
        if chunks is not None:
            assert c.read_tile_size(c.tile_batch) == SUB_TILE_C5 * chunks, "the update ran at another tile size than the one under test"
    finally:
        c.close()


FORCED_SUB_TILES = (2, 3, 4)


def at_tile_sizes(argnames, values, ids=None, forced_values=()):
    """`pytest.mark.parametrize` of a test taking `tiled_ctx` and `argnames`: each of `values` runs under its usual id
    with the slab-size rule, then again at 2, 3 and 4 forced sub-tiles under `<id>-<n>sub`, as do `forced_values`."""
    names = [n.strip() for n in argnames.split(",")]
    as_tuple = (lambda v: tuple(v)) if len(names) > 1 else (lambda v: (v,))
    auto = lambda v: "-".join(str(x) for x in as_tuple(v))  # noqa: E731  (pytest's own ids for ints and strings)
    ids = list(ids) if ids is not None else [auto(v) for v in values]
    params = [pytest.param(None, *as_tuple(v), id=i) for v, i in zip(values, ids)]
    for chunks in FORCED_SUB_TILES:
        params += [pytest.param(chunks, *as_tuple(v), id=f"{i}-{chunks}sub") for v, i in zip(values, ids)]
        params += [pytest.param(chunks, *as_tuple(v), id=f"{auto(v)}-{chunks}sub") for v in forced_values]
    return pytest.mark.parametrize(["tiled_ctx"] + names, params, indirect=["tiled_ctx"])


def sorted_slots(entries: np.ndarray, capacity: int) -> np.ndarray:
    """np.sort(entries) for an alive list: distinct slots below `capacity`, in O(capacity) through a presence mask. A list
    that is not such a set (a test may hand one in) is sorted by np.sort."""
    if len(entries) and int(entries.max()) < capacity:
        mask = np.zeros(capacity, dtype=bool)
        mask[entries] = True
        out = np.flatnonzero(mask).astype(np.uint32)
        if len(out) == len(entries):
            return out
    return np.sort(entries)


@dataclass
class Instance:
    slab_offset: int
    capacity: int
    alive: int = 0          # initial alive count (rows [0, alive) of the alive list are the identity)
    seed: int = 0
    spawn: int = 0


class RefWorld:
    """Oracle-side state of one slab in reference layouts (AoS particles, interleaved indirect rows)."""

    # C5 bodies only (records of 8 words): oracle_update runs orc_update_c5_parallel once per instance of the batch, in batch
    # order, on `parallel_c5` threads, instead of the serial orc_update (same results: test_churn_oracle_cpu.py). A class
    # default, so that tables built without __init__ (object.__new__) have it too.
    parallel_c5 = 0

    def __init__(self, slab_rows: int, stride_words: int, instances: Sequence[Instance], batches: Sequence[Sequence[int]] | None = None,
                 dt: float = 1.0 / 60.0):
        self.slab_rows = slab_rows
        self.stride_words = stride_words
        # HNB_EFFECT_SLOT_ORDER: the update pass visits each instance's particles in ascending particle index — the reference's
        # update when its alive list happens to be sorted. The oracle then reads the list through a sorted copy.
        self.slot_order = False
        self.instances = list(instances)
        n = len(self.instances)
        self.particles = np.zeros((slab_rows, stride_words), dtype=np.uint32)
        self.indirect = np.zeros((slab_rows, 3), dtype=np.uint32)
        self.indirect[:, 2] = np.arange(slab_rows, dtype=np.uint32)  # dead[i] = i (effect_cache.rs:317-319)
        self.metadata = (O.EffectMetadata * n)()
        self.draw = np.zeros(n * 5, dtype=np.uint32)
        self.spawners = (O.Spawner * n)()
        self.prefix = np.zeros(n, dtype=np.uint32)
        self.sim = O.SimParams(dt, 0.0, dt, 0.0, dt, 0.0, n)
        if batches is None:
            batches = [list(range(n))]
        self.batches = [list(b) for b in batches]
        self.batch_infos = (O.BatchInfo * len(self.batches))()
        self.dispatch = np.zeros(3 * len(self.batches), dtype=np.uint32)
        for i, inst in enumerate(self.instances):
            m = self.metadata[i]
            m.capacity = inst.capacity
            m.alive_count = inst.alive
            m.max_update = 0
            m.max_spawn = inst.capacity - inst.alive
            m.indirect_write_index = 0
            m.indirect_render_index = i
            for f in ("init_indirect_dispatch_index", "properties_array_index", "local_child_index", "global_child_index",
                      "base_child_index", "sort_key_offset", "sort_key2_offset"):
                setattr(m, f, 0xFFFFFFFF)
            m.particle_stride = stride_words
            s = self.spawners[i]
            s.transform = O.identity_rows()
            s.inverse_transform = O.identity_rows()
            s.spawn = inst.spawn
            s.seed = inst.seed
            s.effect_metadata_index = i
            s.draw_indirect_index = i
            s.slab_offset = inst.slab_offset
            s.parent_slab_offset = 0xFFFFFFFF
            # alive rows: identity in both ping and pong; dead stack rows [alive, capacity)
            rows = np.arange(inst.alive, dtype=np.uint32)
            self.indirect[inst.slab_offset:inst.slab_offset + inst.alive, 0] = rows
            self.indirect[inst.slab_offset:inst.slab_offset + inst.alive, 1] = rows
        self._rebuild_batches()

    def _rebuild_batches(self):
        """Batcher::push (batch.rs:348-386): CPU prefix sums of the per-instance spawn counts."""
        pos = 0
        for b, members in enumerate(self.batches):
            bi = self.batch_infos[b]
            first = members[0]
            assert members == list(range(first, first + len(members))), "batch members must be consecutive instances"
            bi.total_spawn_count = 0
            bi.total_update_count = 0
            bi.spawner_base = first
            bi.base_particle = self.instances[first].slab_offset
            bi.prefix_sum_offset = first
            bi.prefix_sum_count = len(members)
            run = 0
            for i in members:
                self.prefix[i] = run
                run += max(0, self.spawners[i].spawn)
            pos += len(members)

    def set_spawns(self, spawns: Sequence[int], seeds: Sequence[int] | None = None):
        for i, n in enumerate(spawns):
            self.spawners[i].spawn = int(n)
            if seeds is not None:
                self.spawners[i].seed = int(seeds[i]) & 0xFFFFFFFF
        self._rebuild_batches()

    def batch_spawn_total(self, b: int) -> int:
        return sum(max(0, self.spawners[i].spawn) for i in self.batches[b])

    # ---- oracle passes -------------------------------------------------------------------------
    def oracle_init(self, orc, body, user, b: int = 0):
        total = self.batch_spawn_total(b)
        if total == 0:
            return
        threads = (total + 63) // 64 * 64
        orc.orc_init(C.byref(self.sim), O.ptr(self.particles), self.stride_words, O.ptr(self.indirect), self.spawners,
                     self.prefix.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(self.batch_infos[b]), self.metadata, threads,
                     body, user)

    def oracle_indirect(self, orc):
        orc.orc_indirect(C.byref(self.sim), self.metadata, self.draw.ctypes.data_as(C.POINTER(C.c_uint32)), self.spawners,
                         self.prefix.ctypes.data_as(C.POINTER(C.c_uint32)), None, 0)

    def oracle_prefix_sum(self, orc):
        orc.orc_prefix_sum(self.batch_infos, len(self.batches), self.prefix.ctypes.data_as(C.POINTER(C.c_uint32)),
                           self.dispatch.ctypes.data_as(C.POINTER(C.c_uint32)))

    def sorted_read_lists(self, b: int = 0):
        """Slot order: sort (in place) the alive list every instance of batch `b` is about to be updated through; returns what
        is needed to put the unsorted entries back afterwards (the device never reorders the list it reads)."""
        saved = []
        for i in self.batches[b]:
            md, sp = self.metadata[i], self.spawners[i]
            col, base, n = 1 - md.indirect_write_index, sp.slab_offset, md.max_update
            saved.append((col, base, n, self.indirect[base:base + n, col].copy()))
            self.indirect[base:base + n, col] = sorted_slots(self.indirect[base:base + n, col], md.capacity)
        return saved

    def restore_read_lists(self, saved):
        for col, base, n, rows in saved:
            self.indirect[base:base + n, col] = rows

    def oracle_update(self, orc, body, user, b: int = 0):
        if self.slot_order:
            saved = self.sorted_read_lists(b)
            try:
                self.slot_order = False
                self.oracle_update(orc, body, user, b)
            finally:
                self.slot_order = True
                self.restore_read_lists(saved)
            return
        if self.parallel_c5:
            u32p = C.POINTER(C.c_uint32)
            for i in self.batches[b]:
                md = self.metadata[i]
                flags = np.empty(max(md.max_update, 1), dtype=np.uint8)
                orc.orc_update_c5_parallel(C.byref(self.sim), self.draw.ctypes.data_as(u32p), O.ptr(self.particles),
                                           O.ptr(self.indirect), C.byref(self.spawners[i]), C.byref(md),
                                           C.cast(user, C.POINTER(C.c_float)), O.ptr(flags), self.parallel_c5)
            return
        threads = int(self.dispatch[3 * b]) * 64  # indirect dispatch: x workgroups of 64 threads
        orc.orc_update(C.byref(self.sim), self.draw.ctypes.data_as(C.POINTER(C.c_uint32)), O.ptr(self.particles),
                       self.stride_words, O.ptr(self.indirect), self.spawners,
                       self.prefix.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(self.batch_infos[b]), self.metadata,
                       threads, body, user)

    def set_sort_keys(self, fields):
        """Ribbon effects: sort_key_offset / sort_key2_offset = word offsets of RIBBON_ID / AGE (mod.rs:6037-6046).
        `fields`: the (name, offset, ...) records of asset.particle_layout()."""
        off = {f.name: f.offset // 4 for f in fields}
        for m in self.metadata:
            m.sort_key_offset = off["ribbon_id"]
            m.sort_key2_offset = off["age"]

    def oracle_sort_ribbons(self, orc, literal: bool | None = None):
        """Passes "hanabi:sort_prefix_sum" + per instance fill / sort / copy (mod.rs:7372-7610). `literal` runs
        the restated insertion sort (O(n^2)); otherwise a stable numpy sort of the same (key, key2) pairs."""
        self.oracle_prefix_sum(orc)  # the reference re-runs vfx_prefix_sum over every batch before sorting
        flat = self.indirect.reshape(-1)
        for i in range(len(self.instances)):
            md, sp = self.metadata[i], self.spawners[i]
            n = md.alive_count
            use_literal = literal if literal is not None else n <= 3000
            if use_literal:
                count = C.c_int32(0)
                pairs = np.zeros((max(n, 1), 3), dtype=np.uint32)
                threads = (n + 63) // 64 * 64
                orc.orc_sort_fill(C.byref(count), O.ptr(pairs), O.ptr(self.particles), O.ptr(flat), C.byref(md), C.byref(sp), threads)
                assert count.value == n
                orc.orc_sort(C.byref(count), O.ptr(pairs))
                orc.orc_sort_copy(O.ptr(flat), O.ptr(pairs), C.byref(md), C.byref(sp), threads)
            else:
                col, base = md.indirect_write_index, sp.slab_offset
                e = self.indirect[base:base + n, col].astype(np.int64)
                key = self.particles[base + e, md.sort_key_offset]
                key2 = self.particles[base + e, md.sort_key2_offset]
                order = np.lexsort((key2, key))  # stable, last key is the primary one
                self.indirect[base:base + n, col] = e[order].astype(np.uint32)

    def oracle_frame(self, orc, update_body, update_user=None, init_body=None, init_user=None):
        """init -> indirect -> prefix sum -> update (simulate(), mod.rs:7025-7370)."""
        if init_body is not None:
            for b in range(len(self.batches)):
                self.oracle_init(orc, init_body, init_user, b)
        self.oracle_indirect(orc)
        self.oracle_prefix_sum(orc)
        for b in range(len(self.batches)):
            self.oracle_update(orc, update_body, update_user, b)

    def metadata_rows(self) -> np.ndarray:
        return np.frombuffer(bytes(self.metadata), dtype=np.uint32).reshape(len(self.instances), 15).copy()


class GpuWorld:
    """The same world on the GPU backend, driven through the C ABI only."""

    def __init__(self, ctx, ref: RefWorld, lowered_effect, property_blobs=None, effect=None, sector_planes=False):
        """`property_blobs`: list (per instance) of serialized Properties records, uploaded at array index =
        instance index; the metadata rows of `ref` must carry the same properties_array_index."""
        import bevy_hanabi_b200._native as N
        from bevy_hanabi_b200 import runtime as R
        self.N, self.R = N, R
        self.ctx = ctx
        self.ref = ref
        self.stride = ref.stride_words * 4
        self.slab = ctx.slab_create(ref.slab_rows, self.stride, sector_planes=sector_planes)
        self.effect = effect if effect is not None else ctx.effect_compile(lowered_effect)  # `effect`: an already registered handle
        for i, blob in enumerate(property_blobs or []):
            ctx.upload_properties(self.effect, i, blob)
        ctx.slab_upload_aos(self.slab, 0, ref.particles)
        ctx.slab_upload_indirect(self.slab, 0, ref.indirect)
        if getattr(lowered_effect, "flags", 0) & N.EFFECT_SLOT_ORDER:  # state came from outside: derive the alive bitmap from the lists
            for i, inst in enumerate(ref.instances):
                ctx.slab_rebuild_alive_bits(self.slab, inst.slab_offset, inst.capacity, ref.metadata[i].indirect_write_index, ref.metadata[i].alive_count)
        for i in range(len(ref.instances)):
            md = N.EffectMetadata.from_buffer_copy(bytes(ref.metadata[i]))
            ctx.metadata_insert(i, md)
            ctx.draw_args_insert(i, N.DrawIndexedIndirectArgs(*[int(x) for x in ref.draw[5 * i:5 * i + 5]]))
        self.push_tables()

    def push_tables(self):
        N, ref, ctx = self.N, self.ref, self.ctx
        n = len(ref.instances)
        sp = (N.Spawner * n).from_buffer_copy(bytes(ref.spawners))
        ctx.upload_spawners_raw(sp, n)
        nb = len(ref.batches)
        bi = (N.BatchInfo * nb).from_buffer_copy(bytes(ref.batch_infos))
        # CPU prefix of spawn counts (the oracle's `prefix` array is rewritten by its indirect pass, so rebuild)
        pre = []
        for members in ref.batches:
            run = 0
            for i in members:
                pre.append(run)
                run += max(0, ref.spawners[i].spawn)
        parr = (N.u32 * n)(*pre)
        ctx.upload_batches_raw(bi, nb, parr, n)
        sim = N.SimParams.from_buffer_copy(bytes(ref.sim))
        self.N.check(self.N.lib.hnb_set_sim_params(ctx._h, C.byref(sim)))

    def launches(self):
        return [self.N.BatchLaunch.make(self.effect, self.slab, b, self.ref.batch_spawn_total(b)) for b in range(len(self.ref.batches))]

    def frame(self):
        self.push_tables()
        self.ctx.simulate(self.launches())

    def pull(self):
        """Read everything back in reference layouts."""
        ctx, ref = self.ctx, self.ref
        ctx.sync()
        n = len(ref.instances)
        out = {
            "particles": ctx.slab_download_aos(self.slab, 0, ref.slab_rows, self.stride),
            "indirect": ctx.slab_download_indirect(self.slab, 0, ref.slab_rows),
            "metadata": np.stack([np.frombuffer(bytes(ctx.read_metadata(i)), dtype=np.uint32) for i in range(n)]),
            "draw": np.concatenate([np.frombuffer(bytes(ctx.read_draw_args(i)), dtype=np.uint32) for i in range(n)]),
            "prefix": np.array(ctx.read_prefix_sum(0, n), dtype=np.uint32),
            "batch_infos": np.stack([np.frombuffer(bytes(ctx.read_batch_info(b)), dtype=np.uint32) for b in range(len(ref.batches))]),
            "dispatch": np.concatenate([np.frombuffer(bytes(ctx.read_dispatch_args(b)), dtype=np.uint32) for b in range(len(ref.batches))]),
            "render_pong": np.array([ctx.read_spawner(i).render_pong for i in range(n)], dtype=np.uint32),
        }
        return out


def assert_world_equal(ref: RefWorld, got: dict, float_words=None, rtol=0.0, what="", float_attrs=None):
    """Bit-exact comparison of every buffer (integer bookkeeping AND particle words). When `float_words`
    (boolean mask over the AoS words) and `float_attrs` ([(first_word, count)] of the fp32 attributes) are given,
    those attributes are compared within rtol (see assert_float_attributes_close) instead."""
    np.testing.assert_array_equal(got["metadata"], ref.metadata_rows(), err_msg=f"{what}: effect metadata")
    np.testing.assert_array_equal(got["draw"], ref.draw, err_msg=f"{what}: draw indirect args")
    np.testing.assert_array_equal(got["prefix"], ref.prefix, err_msg=f"{what}: prefix sums")
    bi = np.frombuffer(bytes(ref.batch_infos), dtype=np.uint32).reshape(len(ref.batches), 6)
    np.testing.assert_array_equal(got["batch_infos"], bi, err_msg=f"{what}: batch infos")
    np.testing.assert_array_equal(got["dispatch"], ref.dispatch, err_msg=f"{what}: update dispatch args")
    rp = np.array([ref.spawners[i].render_indirect_read_index for i in range(len(ref.instances))], dtype=np.uint32)
    np.testing.assert_array_equal(got["render_pong"], rp, err_msg=f"{what}: spawner.render_pong")
    np.testing.assert_array_equal(got["indirect"], ref.indirect, err_msg=f"{what}: indirect buffer (ping/pong/dead)")
    if float_words is None or rtol == 0.0:
        np.testing.assert_array_equal(got["particles"], ref.particles, err_msg=f"{what}: particle buffer")
    else:
        fw = np.asarray(float_words, dtype=bool)
        np.testing.assert_array_equal(got["particles"][:, ~fw], ref.particles[:, ~fw], err_msg=f"{what}: particle integer words")
        assert_float_attributes_close(got["particles"], ref.particles, float_attrs, rtol, what)


def float_word_mask(asset):
    """(boolean mask over the AoS words, [(first_word, component_count)] of the fp32 attributes)"""
    from bevy_hanabi_b200 import graph as G
    fields, size, _ = asset.particle_layout()
    mask = np.zeros(size // 4, dtype=bool)
    attrs = []
    for f in fields:
        if not f.name.startswith("pad") and G.vt_elem(f.vt) == "f":
            mask[f.offset // 4: f.offset // 4 + G.vt_count(f.vt)] = True
            attrs.append((f.offset // 4, G.vt_count(f.vt)))
    return mask, attrs


def assert_relaxed_equal(ref: RefWorld, got: dict, what=""):
    """RELAXED_ORDER: counts exact, lists equal as sets per segment, particles identical."""
    np.testing.assert_array_equal(got["metadata"], ref.metadata_rows(), err_msg=f"{what}: effect metadata")
    np.testing.assert_array_equal(got["draw"], ref.draw, err_msg=f"{what}: draw indirect args")
    for i, inst in enumerate(ref.instances):
        md = ref.metadata[i]
        base, alive, W = inst.slab_offset, md.alive_count, md.indirect_write_index
        assert sorted(got["indirect"][base:base + alive, W].tolist()) == sorted(ref.indirect[base:base + alive, W].tolist()), f"{what}: alive set"
        assert sorted(got["indirect"][base + alive:base + inst.capacity, 2].tolist()) == sorted(ref.indirect[base + alive:base + inst.capacity, 2].tolist()), f"{what}: dead set"
    np.testing.assert_array_equal(got["particles"], ref.particles, err_msg=f"{what}: particle buffer")


def assert_ribbons_sorted(ref: RefWorld):
    """Every instance's alive list is in ascending (RIBBON_ID, AGE bits) order."""
    for i in range(len(ref.instances)):
        md, base = ref.metadata[i], ref.spawners[i].slab_offset
        e = ref.indirect[base:base + md.alive_count, md.indirect_write_index].astype(np.int64)
        k = (ref.particles[base + e, md.sort_key_offset].astype(np.uint64) << np.uint64(32)) | ref.particles[base + e, md.sort_key2_offset]
        assert np.all(k[1:] >= k[:-1])


def assert_float_attributes_close(got_words, ref_words, float_attrs, rtol, what=""):
    """"fp32 attributes within `rtol` relative": the error of each component is measured against the magnitude of
    the ATTRIBUTE it belongs to (the largest component of that vector in that particle), so that a component that
    happens to be near zero (cos near pi/2 ...) is not held to an absolute precision fp32 cannot deliver.
    `float_attrs` = [(first_word, component_count), ...]."""
    for first, cnt in float_attrs:
        a = np.ascontiguousarray(got_words[:, first:first + cnt]).view(np.float32)
        b = np.ascontiguousarray(ref_words[:, first:first + cnt]).view(np.float32)
        scale = np.max(np.abs(b), axis=1, keepdims=True)
        err = np.abs(a.astype(np.float64) - b.astype(np.float64))
        bound = rtol * scale.astype(np.float64) + 1e-7
        bad = ~(err <= bound) & ~(np.isnan(a) & np.isnan(b))
        if bad.any():
            i = np.argwhere(bad)[0]
            raise AssertionError(f"{what}: float attribute at words [{first},{first + cnt}): {bad.sum()} components exceed rtol={rtol}; "
                                 f"first at row {i[0]}: got {a[i[0]]} want {b[i[0]]}")


# ---- the lock-step runner ---------------------------------------------------------------------------------------------
def seeds(n, f):
    """Per-instance spawner seeds of frame `f`."""
    return [int(s) for s in pcg_hash(np.arange(n, dtype=np.uint32) + np.uint32(100 * f + 7))]


def is_identity(ref: RefWorld, i: int) -> bool:
    """Whether instance i's current alive list is 0, 1, 2, ..."""
    md, base = ref.metadata[i], ref.instances[i].slab_offset
    lst = ref.indirect[base:base + md.alive_count, md.indirect_write_index]
    return bool((lst == np.arange(len(lst))).all())


class Lockstep:
    """A GpuWorld and the oracle world it must equal, stepped frame by frame and compared after every frame.

    `asset`: an authored effect, stepped by the numpy interpreter with the per-instance property records `props`. Without
    it the world runs C5 under the C oracle's update body with ACCEL_DRAG, on the device the hand-lowered recipes.c5_lowered
    or `effect`, an already compiled C5 module (the authored recipes.c5_asset); `init` adds the constant init of c5_init().
    `relaxed`: lists and dead stacks are compared as sets, then the oracle adopts the device's lists
    (the next frame reads them in the order the device wrote them). `rtol`: fp32 attributes within `rtol` of their
    magnitude, and the device restarts every compared frame from the oracle's records (the bound is a per-step bound:
    libm-level differences are amplified from frame to frame by non-smooth dynamics). `seeds(n, f)`: the spawner seeds of
    frame f, or None to keep them."""

    def __init__(self, ctx, orc, ref, asset=None, *, props=None, init=False, sector=False, slot=False, relaxed=False,
                 fast_math=False, rtol=0.0, seeds=None, effect=None):
        from bevy_hanabi_b200 import recipes
        from oracle.hanabi_oracle import EffectOracle
        from tests.effects import ACCEL_DRAG, c5_init
        self.ctx, self.orc, self.ref, self.slot, self.relaxed, self.rtol, self.seeds = ctx, orc, ref, slot, relaxed, rtol, seeds
        self.fresh, self.got = True, None
        ref.slot_order = slot
        blobs = None
        if asset is None:
            self.eo = None
            self.c_args = [orc.orc_body_update_c5(), ACCEL_DRAG]
            if init:
                self.init = c5_init()  # kept alive: the oracle reads it through a pointer
                self.c_args += [orc.orc_body_init_const(), C.byref(self.init)]
            lowered = recipes.c5_lowered(relaxed_order=relaxed, slot_order=slot)
            self.mask, self.float_attrs = None, None
        else:
            if props is not None:
                blobs = [asset.serialize_properties(p) for p in props]
                for i in range(len(ref.instances)):
                    ref.metadata[i].properties_array_index = i
            self.eo = EffectOracle(asset, dict(enumerate(props)) if props else None)
            lowered = asset.generate(sector_planes=sector, slot_order=slot, relaxed_order=relaxed, fast_math=fast_math)
            self.mask, self.float_attrs = float_word_mask(asset)
        self.gpu = GpuWorld(ctx, ref, lowered, property_blobs=blobs, sector_planes=sector, effect=effect)

    def step(self, f, spawns=None):
        """Frame `f` on both sides, without a comparison. `spawns`: per instance, or None to keep the spawn counts."""
        ref = self.ref
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.sim.virtual_time = ref.sim.real_time = ref.sim.time
        if spawns is not None:
            ref.set_spawns(spawns, self.seeds(len(spawns), f) if self.seeds else None)
        if self.eo is not None:
            self.eo.frame(ref, self.orc)
        else:
            ref.oracle_frame(self.orc, *self.c_args)
        self.gpu.frame()
        self.fresh = False

    def run(self, schedule, start=0, what="", check_every=1):
        """Frames start, start + 1, ... with the spawns of `schedule` (a list of per-instance lists, or a frame count to keep
        the spawn counts), compared after every `check_every`-th and the last. Returns the last pulled state."""
        schedule = [None] * schedule if isinstance(schedule, int) else schedule
        for k, spawns in enumerate(schedule):
            self.step(start + k, spawns)
            if k % check_every == 0 or k == len(schedule) - 1:
                self.compare(f"{what} frame {start + k}")
        return self.got

    def compare(self, what=""):
        ctx, ref, gpu = self.ctx, self.ref, self.gpu
        if self.fresh:  # no frame ran yet: the context has no per-frame tables of this world to read back
            n = len(ref.instances)
            ctx.sync()
            got = {"particles": ctx.slab_download_aos(gpu.slab, 0, ref.slab_rows, gpu.stride),
                   "indirect": ctx.slab_download_indirect(gpu.slab, 0, ref.slab_rows),
                   "metadata": np.stack([np.frombuffer(bytes(ctx.read_metadata(i)), dtype=np.uint32) for i in range(n)]),
                   "draw": np.concatenate([np.frombuffer(bytes(ctx.read_draw_args(i)), dtype=np.uint32) for i in range(n)])}
            for k, want in (("particles", ref.particles), ("indirect", ref.indirect), ("metadata", ref.metadata_rows()), ("draw", ref.draw)):
                np.testing.assert_array_equal(got[k], want, err_msg=f"{what}: {k}")
        else:
            got = gpu.pull()
            if self.relaxed:
                assert_relaxed_equal(ref, got, what)
                ref.indirect[:, :] = got["indirect"]
            else:
                assert_world_equal(ref, got, float_words=self.mask if self.rtol else None, rtol=self.rtol, what=what,
                                   float_attrs=self.float_attrs)
                if self.rtol:
                    ctx.slab_upload_aos(gpu.slab, 0, ref.particles)
        if self.slot:
            assert ctx.read_debug(False)[15] == 0, f"{what}: alive bitmap and counters disagree"
        self.got = got
        return got

    def span(self, i):
        inst = self.ref.instances[i]
        return inst.slab_offset, inst.capacity


# ---- worlds -----------------------------------------------------------------------------------------------------------
def sparks_world(caps, dt=0.05, batches=None, seed=1):
    """Instances of drifting_sparks with capacities `caps`, back to back, none alive, every dead stack shuffled."""
    from tests.effects import drifting_sparks
    asset = drifting_sparks(max(caps))
    _, size, _ = asset.particle_layout()
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=11 + 7 * i))
        off += c
    ref = RefWorld(off, size // 4, insts, batches=batches, dt=dt)
    rng = np.random.default_rng(seed)
    for inst in insts:
        rows = slice(inst.slab_offset, inst.slab_offset + inst.capacity)
        ref.indirect[rows, 2] = rng.permutation(ref.indirect[rows, 2])
    return asset, ref


def table_world(name, caps, batches=None, align=1, dead_perm_seed=None):
    """A slab of instances of tests.effects.EFFECTS[name] with the given capacities, none alive, every dead stack
    shuffled, per-instance emitter translations."""
    from tests.effects import EFFECTS
    _, size, dt, _ = EFFECTS[name]
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


def filled_c5(ctx, orc, insts, fills, batches=None, dead_perm_seed=None, parities=None, effect=None):
    """A Lockstep of C5 with its init over `insts`. `fills`: (first, count, seed, lifetime_lo, lifetime_hi) ranges filled
    by hnb_slab_fill_c5 on the device and orc_fill_c5 in the oracle, after the world was uploaded; the last fill holds the
    claim. `parities`: the alive-list column each instance's first frame appends to (metadata indirect_write_index).
    `effect`: the compiled C5 module the device runs (Lockstep's)."""
    ref = RefWorld(sum(i.capacity for i in insts), 8, insts, batches=batches)
    for i, parity in enumerate(parities or []):
        ref.metadata[i].indirect_write_index = parity
    if dead_perm_seed is not None:  # a dead stack whose slots are not in row order: spawns then append non-identity entries
        rng = np.random.default_rng(dead_perm_seed)
        for inst in insts:
            rows = slice(inst.slab_offset + inst.alive, inst.slab_offset + inst.capacity)
            ref.indirect[rows, 2] = rng.permutation(ref.indirect[rows, 2])
    lock = Lockstep(ctx, orc, ref, init=True, effect=effect)
    for first, count, seed, lo, hi in fills:
        orc.orc_fill_c5(O.ptr(ref.particles), O.ptr(ref.indirect), first, count, seed, lo, hi)
        ctx.slab_fill_c5(lock.gpu.slab, first, count, seed, lo, hi)
    return lock


# Where an identity claim ends, with S = rows per tile: inside or at the end of a warp's 32 rows, of a 128-row sub-tile,
# of a tile.
CLAIM_ENDS = [0, 1, 31, 32, 33, 127, 128, 129, "S-1", "S", "S+1", "3S+17"]
# Spawns per frame: a frame that keeps the claim, a burst that shrinks it to the alive count L, the frame whose write
# column is claimed only up to L (particle L-1 dies in it), two frames without deaths, four frames in which every other
# filled particle dies, and a burst into the freed slots.
CLAIM_EDGE_SPAWNS = [0, 600, 0, 0, 0, 0, 0, 0, 0, 400, 0]


def claim_end(end, S):
    return {"S-1": S - 1, "S": S, "S+1": S + 1, "3S+17": 3 * S + 17}.get(end, end)


def claim_edge_world(L, cap):
    """One C5 instance of `cap` rows, L of them alive, with both alive lists the identity over the whole capacity (as
    hnb_slab_fill_c5 leaves them, with a claim on all `cap` rows). The dead stack hands out slot L+1 first and slot L
    second, the rest shuffled: after the burst, list rows L and L+1 hold slots L+1 and L. Particle L-1 dies in the frame
    after the burst, so the survivor at rank L is slot L while the write column's claim ends at L and its row L still holds
    L+1; every other filled particle dies in frames 5-8 (dt = 1/60)."""
    rng = np.random.default_rng(L)
    ref = RefWorld(cap, 8, [Instance(0, cap, alive=L, seed=31)])
    dt = float(ref.sim.delta_time)
    ref.indirect[:, 0] = ref.indirect[:, 1] = np.arange(cap, dtype=np.uint32)
    ref.indirect[L:, 2] = np.concatenate([[L + 1, L], rng.permutation(np.arange(L + 2, cap))]).astype(np.uint32)
    p = np.zeros((cap, 8), dtype=np.float32)
    p[:, 0:3] = rng.uniform(-1, 1, (cap, 3))
    p[:, 4:7] = rng.uniform(-1, 1, (cap, 3))
    p[:, 7] = rng.uniform(5.5 * dt, 9.0 * dt, cap)
    if L:
        p[L - 1, 7] = 2.5 * dt
    ref.particles[:] = p.view(np.uint32)
    return ref


def claim_edge_lockstep(ctx, orc, L, cap):
    """claim_edge_world on the device: identity lists with a claim on all rows under the scenario's records (writing
    records keeps the claim)."""
    lock = Lockstep(ctx, orc, claim_edge_world(L, cap), init=True)
    ctx.slab_fill_c5(lock.gpu.slab, 0, cap, 1, 1e9, 1e9)
    ctx.slab_upload_aos(lock.gpu.slab, 0, lock.ref.particles)
    return lock


def assert_claims_trusted(lock, n, f):
    """While both alive-list columns of instance 0 are claimed over [0, n), overwrite those rows through the device view
    with two different permutations (in range: a load of them stays in bounds and shows up as a mismatch) and run frame f
    without spawns. The claimed rows must be read as their own index and the stores skipped: both permutations survive,
    and with the identity put back where they stand, every buffer equals the oracle."""
    ctx, ref, gpu = lock.ctx, lock.ref, lock.gpu
    rng = np.random.default_rng(77)
    poison = [rng.permutation(n).astype(np.uint32) for _ in range(2)]
    view = ctx.slab_device_view(gpu.slab)
    ctx.sync()
    for col, ptr in enumerate((view.ping, view.pong)):
        ctx.device_upload(ptr, poison[col])  # not supported for users: done here to observe the claim
    read = ref.metadata[0].indirect_write_index  # the column the next frame reads
    lock.step(f, [0])
    got = gpu.pull()
    np.testing.assert_array_equal(got["indirect"][:n, 1 - read], poison[1 - read], err_msg="claimed stores were not skipped")
    np.testing.assert_array_equal(got["indirect"][:n, read], poison[read], err_msg="the read column was written")
    got["indirect"][:n, :2] = ref.indirect[:n, :2]
    assert_world_equal(ref, got, what="claimed entries were loaded")


# ---- GPU spawn events -------------------------------------------------------------------------------------------------
def oracle_child_init(child, co, cw, po, pw, events, n_valid, seed_c):
    """Child init from GPU spawn events (vfx_init.wgsl:123-171): one thread per event, capped by max_spawn; reads
    the parent particle the event names. Returns the number of children spawned."""
    from oracle.hanabi_oracle import Env, Rng, Writer, apply_modifier
    md = cw.metadata[0]
    n = min(n_valid, md.max_spawn)
    if not n:
        return 0
    k = np.arange(n, dtype=np.int64)
    alive_index = md.alive_count + k
    slots = cw.indirect[alive_index, 2].astype(np.int64)
    pidx = slots.astype(np.uint32)
    parent_idx = events[:n].astype(np.uint32)
    parent_rec = po.unpack(pw.particles[parent_idx.astype(np.int64)].copy())
    rec = np.zeros((n, co.stride_words), dtype=np.uint32)
    P = co.unpack(rec)
    env = Env(n, P, cw.sim, Rng(pcg_hash(pidx ^ np.uint32(seed_c))), {}, pidx, (md.particle_counter + k).astype(np.uint32),
              np.array(list(cw.spawners[0].transform), dtype=np.float32).reshape(3, 4), parent=parent_rec, parent_particle_index=parent_idx)
    wr = Writer()
    for m in child.init_modifiers:
        apply_modifier(m, child.module, env, wr)
    co.pack(P, rec)
    cw.indirect[alive_index, md.indirect_write_index] = pidx
    cw.particles[pidx.astype(np.int64)] = rec
    md.alive_count += n
    md.particle_counter += n
    return n


def oracle_append_events(pw, counts, events, event_count):
    """append_spawn_events_N in serial thread order (lib.rs:976-993); returns the new event_count."""
    from tests.effects import EVENT_CAP
    pidx_rows = pw.indirect[:pw.metadata[0].max_update, 1 - pw.metadata[0].indirect_write_index]
    for row in np.nonzero(counts)[0]:
        c = int(counts[row])
        base = min(event_count, EVENT_CAP)
        event_count += c
        capped = min(c, EVENT_CAP - base)
        events[base:base + capped] = pidx_rows[row]
    return event_count


def emitter_scene(ctx, orc, pcap, ordered):
    """tests.effects.emitter_assets(pcap) for 20 frames: each child consumes its own buffer the frame after. Children come
    BEFORE the parent in batch order, as EffectSorter places them (batch.rs:599-603), so a child's init reads the parent's
    records before the parent's init recycles slots. Without `ordered`, the order in which events land depends on atomic
    scheduling: the buffers are compared as multisets (sub-multisets of what was emitted on overflow) and the oracle
    consumes them in the device's order. With HNB_EFFECT_ORDERED_EVENTS the buffers must hold exactly the canonical
    sequence, overflow included. Every other buffer is compared exactly after every frame."""
    from collections import Counter

    from bevy_hanabi_b200 import _native as N
    from bevy_hanabi_b200 import runtime as R
    from oracle.hanabi_oracle import EffectOracle
    from tests.effects import EVENT_CAP, emitter_assets
    parent, children = emitter_assets(pcap)
    p_fx = parent.generate(num_event_bindings=2, ordered_events=ordered)
    c_fx = [c.generate(parent=parent) for c in children]
    p_stride, c_stride = p_fx.particle_stride, c_fx[0].particle_stride
    dt = 1.0 / 30.0
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
            if ordered:
                np.testing.assert_array_equal(got[:nv], events[k][:nv], err_msg=f"frame {f} channel {k}: event order")
            elif event_count[k] <= EVENT_CAP:
                assert sorted(got[:nv].tolist()) == sorted(events[k][:nv].tolist())
            else:
                # overflow: WHICH appends hit the cap depends on atomic order (lib.rs:980-986), on the reference too;
                # what is defined is that the buffer is full of events that were really emitted
                emitted, kept = Counter(all_emitted[k]), Counter(got.tolist())
                assert all(kept[p] <= emitted[p] for p in kept), f"frame {f} channel {k}: event that nobody emitted"
            events[k][:nv] = got[:nv]   # consume in the GPU buffer's order (the reference's order is unspecified)
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
            spawned[k] += oracle_child_init(children[k], co[k], cw[k], po, pw, events[k], n_valid[k], seed_c[k])
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
            event_count[channel] = oracle_append_events(pw, counts, events[channel], event_count[channel])
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
