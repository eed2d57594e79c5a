"""Ribbon sort (SURVEY.md §8f-4): after the update pass the reference sorts every ribbon effect's alive list by
(RIBBON_ID, AGE bits) — vfx_sort_fill.wgsl, vfx_sort.wgsl (single-thread insertion sort), vfx_sort_copy.wgsl,
driven by simulate() (mod.rs:7372-7610). The CUDA backend does the same stable sort with a shared-memory
bitonic network (n <= 2048) or a cooperative LSD radix sort; both must reproduce the canonical result
(stable with respect to the alive list's canonical order) bit for bit."""
import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import runtime as R
from oracle.hanabi_oracle import EffectOracle
from tests.effects import ribbon_asset
from tests.helpers import GpuWorld, Instance, RefWorld, assert_ribbons_sorted, assert_world_equal

pytestmark = pytest.mark.gpu


def test_ribbon_effect_frames(ctx, orc):
    """Whole frames through hnb_simulate: spawns, deaths, slot recycling, and the sorted alive list every frame."""
    asset = ribbon_asset(4096)
    fx = asset.generate()
    assert fx.flags & N.EFFECT_RIBBONS
    fields, size, _ = asset.particle_layout()
    ref = RefWorld(4096, size // 4, [Instance(0, 4096, alive=0, seed=3)], dt=1 / 30)
    ref.set_sort_keys(fields)
    eo = EffectOracle(asset)
    gpu = GpuWorld(ctx, ref, fx)
    grew_past_small = False
    for f in range(24):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns([900 if f % 4 == 0 else 23])
        eo.frame(ref, orc)
        gpu.frame()
        assert_ribbons_sorted(ref)
        assert_world_equal(ref, gpu.pull(), what=f"frame {f}")
        grew_past_small |= ref.metadata[0].alive_count > 2048
    assert grew_past_small, "the scenario must cross from the shared-memory path to the radix path"


def test_many_ribbon_instances_in_one_batch(ctx, orc):
    """One batch, instances of very different sizes (empty, 1, small, > 2048): one small-path launch covers the
    small ones, the cooperative kernel loops over the large ones."""
    caps = [64, 5000, 1, 300, 2048, 7000, 2, 2100]
    spawn0 = [0, 4200, 1, 250, 2048, 6500, 2, 2100]
    asset = ribbon_asset(sum(caps), ribbons=40.0, lifetime=(0.1, 1.0))
    fx = asset.generate()
    fields, size, _ = asset.particle_layout()
    insts, off = [], 0
    for i, c in enumerate(caps):
        insts.append(Instance(off, c, alive=0, seed=100 + i))
        off += c
    ref = RefWorld(off, size // 4, insts, dt=1 / 30)
    ref.set_sort_keys(fields)
    eo = EffectOracle(asset)
    gpu = GpuWorld(ctx, ref, fx)
    for f in range(8):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        ref.set_spawns(spawn0 if f == 0 else [3, 40, 0, 5, 9, 80, 0, 11])
        eo.frame(ref, orc)
        gpu.frame()
        assert_ribbons_sorted(ref)
        assert_world_equal(ref, gpu.pull(), what=f"frame {f}")


@pytest.mark.parametrize("n", [0, 1, 2, 3, 100, 1000, 2047, 2048, 2049, 5000, 70000, 1 << 20])
@pytest.mark.parametrize("wide_keys", [False, True])
def test_sort_pass_alone(ctx, n, wide_keys):
    """hnb_pass_sort on hand-made state. `wide_keys`: ribbon ids use all 32 bits and ages all exponents, so that
    all eight radix passes run; otherwise few distinct keys, i.e. many ties (stability) and skipped passes."""
    rng = np.random.default_rng(n * 2 + int(wide_keys))
    asset = ribbon_asset(max(n, 1))
    fx = asset.generate()
    fields, size, _ = asset.particle_layout()
    off = {f.name: f.offset // 4 for f in fields}
    words = size // 4
    cap = max(n + 37, 64)
    base = 16                                  # the instance does not start at slab row 0
    slab = ctx.slab_create(base + cap, size)
    effect = ctx.effect_compile(fx)
    particles = rng.integers(0, 2**32, (base + cap, words), dtype=np.uint32)
    if wide_keys:
        particles[:, off["ribbon_id"]] = rng.integers(0, 2**32, base + cap, dtype=np.uint32)
        particles[:, off["age"]] = rng.integers(0, 2**32, base + cap, dtype=np.uint32)
    else:
        particles[:, off["ribbon_id"]] = rng.integers(0, 3, base + cap, dtype=np.uint32)
        particles[:, off["age"]] = rng.choice(np.array([0.0, 0.25, 0.5, 1.5], dtype=np.float32), base + cap).view(np.uint32)
    ctx.slab_upload_aos(slab, 0, particles)
    for col in (0, 1):
        ind = rng.integers(0, 2**32, (base + cap, 3), dtype=np.uint32)     # junk everywhere else: must stay untouched
        perm = rng.permutation(cap)[:n].astype(np.uint32)                  # alive list: distinct slots of the instance
        ind[base:base + n, col] = perm
        ctx.slab_upload_indirect(slab, 0, ind)
        md = R.initial_metadata(cap, 0, words)
        md.alive_count = n
        md.indirect_write_index = col
        md.sort_key_offset, md.sort_key2_offset = off["ribbon_id"], off["age"]
        ctx.metadata_insert(0, md)
        ctx.draw_args_insert(0)
        ctx.upload_spawners([R.make_spawner(slab_offset=base)])
        ctx.upload_batches([N.BatchInfo(0, 0, 0, base, 0, 1)], [0])
        ctx.set_sim_params(1 / 60, 0.0, 1)
        ctx.pass_sort(N.BatchLaunch.make(effect, slab, 0, 0))
        got = ctx.slab_download_indirect(slab, 0, base + cap)
        e = perm.astype(np.int64)
        order = np.lexsort((particles[base + e, off["age"]], particles[base + e, off["ribbon_id"]]))
        want = ind.copy()
        want[base:base + n, col] = perm[order]
        np.testing.assert_array_equal(got, want, err_msg=f"n={n} column {col}")
    np.testing.assert_array_equal(ctx.slab_download_aos(slab, 0, base + cap, size), particles)
