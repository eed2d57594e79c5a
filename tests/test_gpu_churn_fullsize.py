"""The 16 Mi-slot churn steady state that tools/perf_matrix.py measures (`_churned`), held to the oracle: 16 Mi slots of
tests.effects.drifting_sparks (its own column plan, lifetime floors and group ages) after 240 frames of P / 40 spawns per
frame into recycled slots, so the alive list is a scattered permutation of the slab, the dead stack is fed by deaths from
thousands of tiles, and the update gathers rows through a persistent grid at the tile size the slab-size rule picks.

The oracle runs the C bodies that tests/test_churn_oracle_cpu.py proves equal to the numpy interpreter: orc_body_init_sparks
and orc_update_c5_parallel. Each trajectory is computed once per module and size. A full pull is 700 MB at 16 Mi, so
after every frame the device is compared through non-flushing or order-independent reads: hnb_slab_checksum of the whole
slab (dead rows included: both sides write them), hnb_slab_checksum_indirect of the interleaved list rows, metadata row 0
and draw-args row 0. After frames 1, 2, 40 and 240, and at the end of each branch, everything is pulled: at frame 240 of
the list-order trajectory it is compared with the oracle's state word for word; elsewhere, where keeping every state would
take gigabytes, each record row and each list row with a 32-bit digest of the oracle's (row index mixed in). A failure
names the first frame that differed and the first differing rows of the next full pull.

Cases, each also at 1 Mi slots (quick to debug):
- the steady state in list order and with sector planes (one oracle trajectory), and in slot order (its own, the oracle
  reading sorted lists), with the scenario's own checks: alive count, particles spawned, how scattered the list is;
- a repack at frame 240 into floor tiles that defer common ages (DESIGN.md §3), then 60 churn frames in which the first
  death ends the claim and gathered tiles consume the deferred words; with only non-flushing reads per frame (`quiet`),
  with record checksums, which flush, per frame (`every`), and with HNB_DEFER_AGES=0 (control);
- bounds, depth order, cull, cull of the depth order and four-view cull of the churned state, which change nothing;
- a snapshot of the churned instance, restored into a second slab, then 20 churn frames there."""
from __future__ import annotations

import time

import numpy as np
import pytest

from oracle import c_oracle as O
from tests.bounds_ref import BOUNDS_DTYPE, assert_bounds_equal, ref_bounds
from tests.cull_ref import ref_cull
from tests.depth_order_ref import ref_depth_order
from tests.effects import ACCEL_DRAG, drifting_sparks, sparks_init
from tests.helpers import GpuWorld, Instance, RefWorld, assert_world_equal
from tests.repack_ref import ref_repack
from tests.snapshot_ref import ref_restore, ref_snapshot

pytestmark = pytest.mark.gpu

DT = 1.0 / 60.0
LIFETIME = (0.2, 0.9)
INIT = sparks_init(LIFETIME)  # kept alive: the oracle reads it through a pointer
FRAMES = 240
FULL = (1, 2, 40, 240)                 # full pulls, after this many frames
REPACK_END, REPACK_FULL = 300, (250, 300)
RESTORE_END = 260
STRIDE_WORDS = 8
SENTINEL = np.uint32(0xA5A5A5A5)
# tools/perf_matrix.py's frusta: x in [0, 2], y and z in [-2, 2] keeps about half of the cloud over [-1, 1]^3; its
# view_frusta(4) turns the first plane around the y axis and tilts it up and down
CULL_HALF = [[1, 0, 0, 0], [-1, 0, 0, 2], [0, 1, 0, 2], [0, -1, 0, 2], [0, 0, 1, 2], [0, 0, -1, 2]]
TIMES = {"oracle": 0.0}


def view_frusta(views):
    out = []
    for v in range(views):
        t = 2 * np.pi * v / max(views, 1)
        n = np.array([np.cos(t), 0.3 * (-1) ** v, np.sin(t)])
        n /= np.linalg.norm(n)
        out.append([[*n, 0.0]] + CULL_HALF[1:])
    return np.array(out, dtype=np.float32)


# ---- oracle side ------------------------------------------------------------------------------------------------------
def new_world(P):
    """One instance of P slots at row 0, nothing alive, the dead stack of a new slab."""
    from oracle.host_threads import oracle_threads
    ref = RefWorld(P, STRIDE_WORDS, [Instance(0, P, alive=0, seed=0)], dt=DT)
    ref.parallel_c5 = oracle_threads()
    return ref


def clone(ref):
    c = RefWorld.__new__(RefWorld)
    c.__dict__.update(ref.__dict__)
    for k in ("particles", "indirect", "draw", "prefix", "dispatch"):
        setattr(c, k, getattr(ref, k).copy())
    for k in ("metadata", "spawners", "batch_infos", "sim"):
        v = getattr(ref, k)
        setattr(c, k, type(v).from_buffer_copy(v))
    c.instances, c.batches = list(ref.instances), [list(b) for b in ref.batches]
    return c


def set_frame(ref, f):
    """Frame f of _churned: P / 40 spawns with seed 1000 + f."""
    ref.sim.time = ref.sim.virtual_time = ref.sim.real_time = np.float32(f) * ref.sim.delta_time
    ref.set_spawns([ref.slab_rows // 40], [1000 + f])


def oracle_frame(orc, ref, f):
    t0 = time.perf_counter()
    set_frame(ref, f)
    ref.oracle_frame(orc, orc.orc_body_update_c5(), ACCEL_DRAG, orc.orc_body_init_sparks(), INIT)
    TIMES["oracle"] += time.perf_counter() - t0


def observe(orc, ref):
    """What the device is compared with after every frame."""
    t0 = time.perf_counter()
    out = {"records": orc.orc_checksum(O.ptr(ref.particles), 0, ref.slab_rows, STRIDE_WORDS),
           "lists": orc.orc_checksum(O.ptr(ref.indirect), 0, ref.slab_rows, 3),
           "metadata": ref.metadata_rows()[0], "draw": ref.draw[:5].copy()}
    TIMES["oracle"] += time.perf_counter() - t0
    return out


def digests(orc, words):
    """A 32-bit digest per row of a (rows, k) uint32 array: the high half of the row's term of orc_checksum."""
    words = np.ascontiguousarray(words, dtype=np.uint32)
    out = np.empty(len(words), dtype=np.uint32)
    orc.orc_row_digests(O.ptr(words), len(words), words.shape[1], O.ptr(out))
    return out


def full_digests(orc, ref):
    t0 = time.perf_counter()
    out = {"records": digests(orc, ref.particles), "lists": digests(orc, ref.indirect), "metadata": ref.metadata_rows()[0],
           "draw": ref.draw[:5].copy()}
    TIMES["oracle"] += time.perf_counter() - t0
    return out


def trajectory(orc, ref, frames, full, keep_last=False):
    """Frames `frames` of `ref`: (per frame count, what the device is compared with), (full digests by frame count)."""
    t0 = time.perf_counter()
    seen, digs = {}, {}
    for f in frames:
        oracle_frame(orc, ref, f)
        seen[f + 1] = observe(orc, ref)
        if f + 1 in full and not (keep_last and f == frames[-1]):
            digs[f + 1] = full_digests(orc, ref)
    return seen, digs, time.perf_counter() - t0


@pytest.fixture(scope="module", autouse=True)
def oracle_share():
    t0, o0 = time.perf_counter(), TIMES["oracle"]
    yield
    total, oracle = time.perf_counter() - t0, TIMES["oracle"] - o0
    print(f"\nchurn full size: {total:.1f} s in all, of which the oracle {oracle:.1f} s ({100 * oracle / max(total, 1e-9):.0f} %)")


@pytest.fixture(scope="module", params=[1 << 20, 16 << 20], ids=["1Mi", "16Mi"])
def size(request):
    return request.param


@pytest.fixture(scope="module")
def churn(size, orc):
    """The list-order trajectory: per-frame observations, digests after frames 1, 2 and 40, and the state after 240."""
    ref = new_world(size)
    seen, digs, s = trajectory(orc, ref, range(FRAMES), FULL, keep_last=True)
    print(f"\noracle: {size >> 20} Mi slots x {FRAMES} frames in list order: {s:.1f} s")
    return {"seen": seen, "full": digs, "ref": ref}


@pytest.fixture(scope="module")
def churn_slot(size, orc):
    ref = new_world(size)
    ref.slot_order = True
    seen, digs, s = trajectory(orc, ref, range(FRAMES), FULL)
    print(f"\noracle: {size >> 20} Mi slots x {FRAMES} frames in slot order: {s:.1f} s")
    return {"seen": seen, "full": digs}


@pytest.fixture(scope="module")
def repacked(churn, orc):
    """Instance 0 repacked after frame 240, then frames 240-299."""
    ref = clone(churn["ref"])
    ref_repack(ref, 0)
    at = observe(orc, ref)
    seen, digs, s = trajectory(orc, ref, range(FRAMES, REPACK_END), REPACK_FULL)
    print(f"\noracle: repack and {REPACK_END - FRAMES} frames: {s:.1f} s")
    return {"repack": at, "seen": seen, "full": digs}


@pytest.fixture(scope="module")
def restored(churn, orc):
    """The snapshot of instance 0 after frame 240 restored into a new slab, then frames 240-259 there."""
    ref = new_world(churn["ref"].slab_rows)
    ref_restore(ref, 0, ref_snapshot(churn["ref"], 0))
    at = observe(orc, ref)
    seen, digs, s = trajectory(orc, ref, range(FRAMES, RESTORE_END), (RESTORE_END,))
    print(f"\noracle: restore and {RESTORE_END - FRAMES} frames: {s:.1f} s")
    return {"restore": at, "seen": seen, "full": digs}


# ---- device side ------------------------------------------------------------------------------------------------------
@pytest.fixture()
def make_ctx(native, monkeypatch):
    """Fresh contexts at the tile size the slab-size rule picks; defer=False: HNB_DEFER_AGES=0."""
    made = []
    monkeypatch.delenv("HNB_TILE_CHUNKS", raising=False)

    def make(defer=True):
        if defer:
            monkeypatch.delenv("HNB_DEFER_AGES", raising=False)
        else:
            monkeypatch.setenv("HNB_DEFER_AGES", "0")
        made.append(native.Context(0))
        return made[-1]
    yield make
    for c in made:
        c.close()


class Device:
    """The device side of a trajectory: a GpuWorld whose RefWorld holds only the per-frame tables (the records live on the
    device), checked after every frame against an oracle trajectory. Mismatches are recorded, not raised, so that the next
    full pull can name the first frame that differed and the rows that differ."""

    def __init__(self, ctx, orc, P, sector=False, slot=False, effect=None, what=""):
        self.ctx, self.orc, self.P, self.slot, self.what = ctx, orc, P, slot, what
        self.fx = drifting_sparks(P).generate(sector_planes=sector, slot_order=slot)
        self.tables = new_world(P)
        self.gpu = GpuWorld(ctx, self.tables, self.fx, sector_planes=sector, effect=effect)
        self.tables.particles = self.tables.indirect = None  # uploaded: the device holds the records from here on
        self.slab, self.first_bad = self.gpu.slab, None

    def frame(self, f):
        set_frame(self.tables, f)
        self.gpu.frame()

    def check(self, label, want, records=True):
        """Compare with an observation of the oracle; `records`: also hnb_slab_checksum (which flushes deferred groups)."""
        ctx, got = self.ctx, {}
        if records:
            got["records"] = ctx.slab_checksum(self.slab, 0, self.P)
        got["lists"] = ctx.slab_checksum_indirect(self.slab, 0, self.P)
        got["metadata"] = np.frombuffer(bytes(ctx.read_metadata(0)), dtype=np.uint32)
        got["draw"] = np.frombuffer(bytes(ctx.read_draw_args(0)), dtype=np.uint32)
        bad = [k for k in got if not np.array_equal(got[k], want[k])]
        if bad and self.first_bad is None:
            self.first_bad = f"{label} ({', '.join(bad)})"
        if self.slot:
            assert ctx.read_debug(False)[15] == 0, f"{self.what} {label}: alive bitmap and counters disagree"

    def run(self, frames, seen, full=()):
        """Frames `frames`, checked after each against seen[count]; a full pull after the frame counts of `full` (each
        digests, or a RefWorld)."""
        for f in frames:
            self.frame(f)
            self.check(f"frame {f + 1}", seen[f + 1])
            if f + 1 in full:
                self.full_compare(f"frame {f + 1}", full[f + 1])

    def full_compare(self, label, want):
        """Everything pulled, against a RefWorld word for word or against digests row by row."""
        got = self.gpu.pull()
        if isinstance(want, RefWorld):
            rec = np.flatnonzero((got["particles"] != want.particles).any(axis=1))
            lst = np.flatnonzero((got["indirect"] != want.indirect).any(axis=1))
        else:
            rec = np.flatnonzero(digests(self.orc, got["particles"]) != want["records"])
            lst = np.flatnonzero(digests(self.orc, got["indirect"]) != want["lists"])
        msg = (f"{self.what}: first frame that differs: {self.first_bad}; at {label}: {len(rec)} record rows differ "
               f"(first {rec[:8].tolist()}), {len(lst)} list rows differ (first {lst[:8].tolist()})")
        assert self.first_bad is None and not len(rec) and not len(lst), msg
        if isinstance(want, RefWorld):
            assert_world_equal(want, got, what=f"{self.what} {label}")
        else:
            np.testing.assert_array_equal(got["metadata"][0], want["metadata"], err_msg=f"{self.what} {label}: metadata")
            np.testing.assert_array_equal(got["draw"][:5], want["draw"], err_msg=f"{self.what} {label}: draw args")
        return got


def steady(ctx, orc, churn, P, what, full=True, **kw):
    """The device through the 240 frames of `churn`; full pulls at FULL, or none (the branches, which start from there)."""
    t0 = time.perf_counter()
    dev = Device(ctx, orc, P, what=what, **kw)
    want = dict(churn["full"])
    if "ref" in churn:
        want[FRAMES] = churn["ref"]
    dev.run(range(FRAMES), churn["seen"], want if full else {})
    print(f"\n{what}: device {time.perf_counter() - t0:.1f} s")
    return dev


def scenario_checks(ctx, dev, P, what):
    """The state is what it claims: a population around 0.8 P, every slot recycled several times, a scattered list."""
    md = ctx.read_metadata(0)
    lst = ctx.slab_download_indirect(dev.slab, 0, 1 << 16)[:, md.indirect_write_index].astype(np.int64)
    jump = float(np.median(np.abs(np.diff(lst))))
    print(f"{what}: {md.alive_count / P:.3f} P alive, {md.particle_counter / P:.2f} P spawned, median |slot jump| {jump:.0f}")
    assert 0.7 * P < md.alive_count < 0.9 * P
    assert md.particle_counter > 3 * P
    assert jump > 1000, "the alive list must be a scattered gather"


@pytest.mark.parametrize("layout", ["default", "sector"])
def test_steady_state(make_ctx, orc, churn, size, layout):
    ctx = make_ctx()
    dev = steady(ctx, orc, churn, size, f"{size >> 20} Mi {layout}", sector=layout == "sector")
    scenario_checks(ctx, dev, size, f"{size >> 20} Mi {layout}")


def test_steady_state_slot_order(make_ctx, orc, churn_slot, size):
    ctx = make_ctx()
    steady(ctx, orc, churn_slot, size, f"{size >> 20} Mi slot order", slot=True)


@pytest.mark.parametrize("mode,defer", [("quiet", True), ("every", True), ("quiet", False)], ids=["quiet", "every", "control"])
def test_repack_into_deferred_ages(make_ctx, orc, churn, repacked, size, mode, defer):
    """Repack after frame 240, then 60 churn frames. `quiet`: per frame only reads that flush nothing (list checksum,
    metadata, deferred count), records at frames 250 and 300; `every`: record checksums every frame as well."""
    ctx = make_ctx(defer)
    what = f"{size >> 20} Mi repack {mode}{'' if defer else ' control'}"
    dev = steady(ctx, orc, churn, size, what, full=False)
    assert "#define HNB_GROUP_AGE 1" in dev.fx.generate_source()
    t0 = time.perf_counter()
    ctx.slab_repack(dev.slab, dev.gpu.effect, 0, 0, size)
    dev.check("the repack", repacked["repack"], records=mode == "every")
    counts = []
    for f in range(FRAMES, REPACK_END):
        dev.frame(f)
        counts.append(ctx.slab_deferred_groups(dev.slab))  # before anything that flushes
        dev.check(f"frame {f + 1}", repacked["seen"][f + 1], records=mode == "every")
        if f + 1 in REPACK_FULL:
            dev.full_compare(f"frame {f + 1}", repacked["full"][f + 1])
    print(f"{what}: device {time.perf_counter() - t0:.1f} s; deferred groups after frames 241..: {counts[:8]} "
          f"(max {max(counts)} of {size // 32})")
    if defer:
        k = next((k for k, n in enumerate(counts) if n), None)
        assert k is not None, "no update after the repack left a group deferred: the case proves nothing"
        assert counts[k + 1] == 0, "the update after a deferring one walks every row of every deferred group"
    else:
        assert max(counts) == 0


def test_batch_passes_on_churned_state(make_ctx, orc, churn, size):
    """Bounds, depth order, cull (of the alive list and of the depth order) and a four-view cull of the churned state after
    frame 240, against the restatements on the oracle's state; the slab, its lists and the tables stay as they were."""
    ctx = make_ctx()
    P, ref = size, churn["ref"]
    dev = steady(ctx, orc, churn, P, f"{P >> 20} Mi batch passes", full=False)
    launch = dev.gpu.launches()[0]
    views = 4
    frusta = np.array([CULL_HALF], dtype=np.float32)
    planes = np.array([[0.36, -0.48, 0.8, 0.05]], dtype=np.float32)
    multi = view_frusta(views)[:, None]  # (views, instances, 6, 4)
    d = {k: ctx.device_alloc(n) for k, n in (("bounds", 32), ("planes", 16), ("frusta", 96), ("multi", 96 * views),
                                              ("order", 4 * P), ("visible", 4 * P), ("visible4", 4 * views * P),
                                              ("args", 20), ("args4", 20 * views))}
    try:
        ctx.device_upload(d["planes"], planes.view(np.uint32))
        ctx.device_upload(d["frusta"], frusta.reshape(-1).view(np.uint32))
        ctx.device_upload(d["multi"], multi.reshape(-1).view(np.uint32))
        fill = np.full(views * P, SENTINEL, dtype=np.uint32)
        for k in ("order", "visible", "visible4"):
            ctx.device_upload(d[k], fill[:(views if k == "visible4" else 1) * P])

        ctx.batch_bounds(launch, d["bounds"], 1)
        got = ctx.device_download(d["bounds"], 32).view(BOUNDS_DTYPE)
        assert_bounds_equal(got, ref_bounds(ref, 0, 0), "bounds")
        assert got["count"][0] == ref.metadata[0].alive_count

        ctx.batch_depth_order(launch, d["planes"], 1, d["order"], P)
        order = ref_depth_order(ref, 0, 0, planes, fill[:P])
        np.testing.assert_array_equal(ctx.device_download(d["order"], 4 * P), order, err_msg="depth order")

        for src, what in ((0, "alive list"), (d["order"], "depth order")):
            ctx.device_upload(d["visible"], fill[:P])
            ctx.batch_cull(launch, d["frusta"], 1, src, P if src else 0, d["visible"], P, d["args"], 1)
            vis, args = ref_cull(ref, 0, 0, frusta, fill[:P], ref.draw, src=order if src else None)
            np.testing.assert_array_equal(ctx.device_download(d["visible"], 4 * P), vis, err_msg=f"cull of the {what}")
            np.testing.assert_array_equal(ctx.device_download(d["args"], 20).reshape(1, 5), args, err_msg=f"cull args, {what}")
            frac = args[0, 1] / ref.metadata[0].alive_count
            print(f"cull of the {what}: {frac:.3f} of the live particles visible")
            assert 0.3 < frac < 0.7

        ctx.batch_cull_views(launch, views, d["multi"], 1, 0, 0, d["visible4"], P, d["args4"], 1)
        vis4 = ctx.device_download(d["visible4"], 4 * views * P).reshape(views, P)
        args4 = ctx.device_download(d["args4"], 20 * views).reshape(views, 1, 5)
        for v in range(views):
            vis, args = ref_cull(ref, 0, 0, multi[v], fill[:P], ref.draw)
            np.testing.assert_array_equal(vis4[v], vis, err_msg=f"cull view {v}")
            np.testing.assert_array_equal(args4[v], args, err_msg=f"cull args, view {v}")
    finally:
        for p in d.values():
            ctx.device_free(p)
    dev.check("the batch passes", churn["seen"][FRAMES])
    assert dev.first_bad is None, f"the batch passes changed the world: {dev.first_bad}"


def test_snapshot_restore_churned(make_ctx, orc, churn, restored, size):
    """A snapshot of the churned instance after frame 240 equals the restatement byte for byte; restored into a second
    slab (a claim on its rows, so the first update runs floor tiles and the next gathered ones), it churns 20 more frames
    as the oracle does."""
    ctx = make_ctx()
    P = size
    dev = steady(ctx, orc, churn, P, f"{P >> 20} Mi snapshot", full=False)
    want = ref_snapshot(churn["ref"], 0)
    nbytes = ctx.instance_snapshot_bytes(4 * STRIDE_WORDS, P)
    d = ctx.device_alloc(nbytes)
    try:
        ctx.instance_snapshot(dev.slab, dev.gpu.effect, 0, 0, P, d, nbytes)
        np.testing.assert_array_equal(ctx.device_download(d, want.nbytes), want, err_msg="snapshot bytes")
        del want
        second = Device(ctx, orc, P, effect=dev.gpu.effect, what=f"{P >> 20} Mi restored")
        ctx.instance_restore(second.slab, second.gpu.effect, 0, 0, P, d, nbytes)
        ctx.sync()
    finally:
        ctx.device_free(d)
    second.check("the restore", restored["restore"])
    counts = []
    for f in range(FRAMES, RESTORE_END):
        second.frame(f)
        counts.append(ctx.slab_deferred_groups(second.slab))
        # records from frame 243 on: hnb_slab_checksum flushes, and the first two frames are the floor tiles and the
        # gathered tiles that meet what they deferred
        second.check(f"frame {f + 1}", restored["seen"][f + 1], records=f >= FRAMES + 2)
        if f + 1 == RESTORE_END:
            second.full_compare(f"frame {f + 1}", restored["full"][f + 1])
    print(f"{P >> 20} Mi restored: deferred groups after frames 241..: {counts[:8]}")
