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

SUB_TILE_C5 = 128  # rows of an update sub-tile for C5 records: 32 lanes x K = 4 rows in flight per lane


@pytest.fixture(params=[1, 2, 3, 4], ids=lambda n: f"{n}sub")
def tiled_ctx(request, native, monkeypatch):
    """A fresh context on cuda:0 whose update tiles hold `tile_chunks` sub-tiles, forced with HNB_TILE_CHUNKS (None: the
    slab-size rule of plan_batch, which picks 1 below one wave of resident warps, about 400 Ki rows for C5, so without the
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


@dataclass
class Instance:
    slab_offset: int
    capacity: int
    alive: int = 0          # initial alive count (rows [0, alive) of the alive list are the identity)
    seed: int = 0
    spawn: int = 0


class RefWorld:
    """Oracle-side state of one slab in reference layouts (AoS particles, interleaved indirect rows)."""

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
            self.indirect[base:base + n, col] = np.sort(self.indirect[base:base + n, col])
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
