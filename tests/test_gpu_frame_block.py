"""The two things that keep a frame a pure kernel chain when the HOST changes its tables every frame (round 2):
  * the frame block (header + every host-written table) travels in the bookkeeping kernel's parameter space instead of through a
    copy-engine operation (frames without an init pass whose tables fit: HNB_FRAME_BLOCK_MAX_BYTES);
  * the count mailbox: the update pass posts (epoch, instance_count) into pinned host memory, so reading a frame's counts needs
    no device-to-host copy and no event.
Both must be invisible in the results: same buffers as the copy path, same counts as the draw-indirect rows."""
import numpy as np
import pytest

from bevy_hanabi_b200 import recipes
from oracle.hanabi_oracle import pcg_hash
from tests.effects import ACCEL_DRAG, fill_c5, firework_trails
from tests.helpers import GpuWorld, Instance, Lockstep, RefWorld, assert_world_equal

pytestmark = pytest.mark.gpu


def _world(batches=None):
    ref = RefWorld(3 * 4096, 8, [Instance(0, 4096, alive=4000, seed=1), Instance(4096, 4096, alive=1, seed=2), Instance(8192, 4096, alive=4096, seed=3)], batches=batches)
    fill_c5(ref, np.random.default_rng(5), 0.02, 0.6)
    return ref


@pytest.mark.parametrize("batches", [None, [[0], [1], [2]], [[0, 1], [2]]])
@pytest.mark.parametrize("param_upload", ["1", "0"])
def test_tables_rewritten_every_frame(native, orc, monkeypatch, param_upload, batches):
    """Three instances in one, three or two batches (= CTAs of the bookkeeping grid: CTA 0 stores the block while the others
    write the device-owned words of their rows), deaths, and a host that re-uploads spawners / batches / sim params EVERY frame (GpuWorld.frame
    does) with new seeds: oracle parity frame by frame on both upload paths; the parameter path performs no frame-block copy."""
    monkeypatch.setenv("HNB_PARAM_UPLOAD", param_upload)
    ctx = native.Context(0)
    ref = _world(batches)
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    frames0, copies0 = ctx.frames_simulated, ctx.frame_block_copies
    for f in range(20):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns([0, 0, 0], [100 + f, 200 + f, 300 + f])
        _oracle_c5_frame(ref, orc)
        gpu.frame()
        assert_world_equal(ref, gpu.pull(), what=f"frame {f} (HNB_PARAM_UPLOAD={param_upload})")
    frames1, copies1 = ctx.frames_simulated, ctx.frame_block_copies
    assert frames1 - frames0 == 20
    assert copies1 - copies0 == (0 if param_upload == "1" else 20)
    assert 0 < ref.metadata[0].alive_count < 4000
    ctx.close()


def _oracle_c5_frame(ref, orc):
    ref.oracle_frame(orc, orc.orc_body_update_c5(), ACCEL_DRAG)


def test_count_mailbox(ctx, orc):
    """The mailbox word of frame `epoch` = that frame's draw-indirect instance_count, for every instance of the batch; two frames
    are kept in flight (the ring has four slots) and a detached mailbox is left alone."""
    ref = _world()
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    box = ctx.set_count_mailbox(rows=3, ring=4)
    epochs = []
    for f in range(12):
        ref.set_spawns([0, 0, 0])
        _oracle_c5_frame(ref, orc)
        gpu.frame()
        epochs.append((ctx.last_epoch(), [int(ref.draw[5 * i + 1]) for i in range(3)]))
        if f >= 1:  # check the PREVIOUS frame while this one is queued
            e, want = epochs[f - 1]
            assert [ctx.mailbox_count(e, i) for i in range(3)] == want
    e, want = epochs[-1]
    assert [ctx.mailbox_count(e, i) for i in range(3)] == want
    assert want == [ctx.read_draw_args(i).instance_count for i in range(3)]
    assert len({e for e, _ in epochs}) == 12 and all(b > a for (a, _), (b, _) in zip(epochs, epochs[1:]))
    ctx.set_count_mailbox(rows=0)
    snapshot = list(box)
    gpu.frame()
    ctx.sync()
    assert list(box) == snapshot


@pytest.mark.parametrize("param_upload", ["1", "0"])
def test_spawns_every_frame(native, orc, monkeypatch, param_upload):
    """Frames WITH an init pass: the block is stored by a one-CTA kernel at the head of the frame (init reads the tables after its
    dependency wait then) — the firework recipe spawning every frame into recycled slots, zero tolerance, on both upload paths."""
    monkeypatch.setenv("HNB_PARAM_UPLOAD", param_upload)
    ctx = native.Context(0)
    asset = firework_trails(4096)
    ref = RefWorld(4096, 12, [Instance(0, 4096, alive=0)], dt=1.0 / 20.0)
    seeds = lambda n, f: [int(pcg_hash(np.array([0x777 + f], dtype=np.uint32))[0])]
    copies0 = ctx.frame_block_copies
    Lockstep(ctx, orc, ref, asset, seeds=seeds).run([[300 if f % 7 else 900] for f in range(60)], check_every=3)
    copies = ctx.frame_block_copies - copies0
    assert (copies == 0) if param_upload == "1" else (copies >= 60)
    assert ref.metadata[0].particle_counter > 3 * 4096, "slots were recycled"
    ctx.close()


@pytest.mark.parametrize("n_inst", [30, 40, 200])
def test_large_parameter_blocks(ctx, orc, n_inst):
    """Tables beyond the classic 4 KB parameter space (30 instances: 4.2 KB, one warp + helper warps for the store; 40: the
    many-instance path; 200: 27 KB) still travel with the launch (CUDA 12.1+: 32 KB of kernel parameters)."""
    cap = 256
    ref = RefWorld(n_inst * cap, 8, [Instance(i * cap, cap, alive=200 + (i % 50), seed=i) for i in range(n_inst)])
    fill_c5(ref, np.random.default_rng(n_inst), 0.02, 0.4)
    gpu = GpuWorld(ctx, ref, recipes.c5_lowered())
    copies0 = ctx.frame_block_copies
    for f in range(8):
        ref.set_spawns([0] * n_inst, [1000 * f + i for i in range(n_inst)])
        _oracle_c5_frame(ref, orc)
        gpu.frame()
        assert_world_equal(ref, gpu.pull(), what=f"{n_inst} instances, frame {f}")
    assert ctx.frame_block_copies == copies0
