"""A whole "scene" through both API levels, frame after frame: several effect assets with different particle
layouts, several instances each, spawn counts from EffectSpawner::tick (spawn.rs:838-921), batches from
Batcher::push (batch.rs:348-386), one hnb_simulate per frame — i.e. what the render thread does with the
reference (prepare_effects -> batch_effects -> simulate, SURVEY.md §3.4). Every asset's slab is compared with its
own oracle world after every frame, bit for bit (all effects here use IEEE-exact operations only).

The multi-batch frame exercises the fork/join of the init and update launches over the context's side streams.
"""
import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import runtime as R
from bevy_hanabi_b200 import spawn as S
from oracle.hanabi_oracle import EffectOracle, pcg_hash
from tests.effects import drifting_sparks, firework_trails, growing_dust, ribbon_asset
from tests.helpers import Instance, RefWorld

pytestmark = pytest.mark.gpu


class SceneEffect:
    def __init__(self, ctx, asset, capacities, settings, first_row, dt):
        self.asset, self.first_row = asset, first_row
        self.fx = asset.generate()
        fields, size, _ = asset.particle_layout()
        insts, off = [], 0
        for c in capacities:
            insts.append(Instance(off, c))
            off += c
        self.ref = RefWorld(off, size // 4, insts, dt=dt)
        self.ribbons = bool(self.fx.flags & N.EFFECT_RIBBONS)
        if self.ribbons:
            self.ref.set_sort_keys(fields)
        self.oracle = EffectOracle(asset)
        self.spawners = [S.EffectSpawner(st, rng_seed=first_row * 977 + i) for i, st in enumerate(settings)]
        self.slab = ctx.slab_create(off, size)
        self.effect = ctx.effect_compile(self.fx)
        self.stride = size
        for i in range(len(insts)):
            md = N.EffectMetadata.from_buffer_copy(bytes(self.ref.metadata[i]))
            md.indirect_draw_index = first_row + i
            ctx.metadata_insert(first_row + i, md)
            ctx.draw_args_insert(first_row + i)


def test_scene_of_four_assets(ctx, orc):
    dt = 1.0 / 60.0
    plan = [
        (firework_trails(1), [3000, 500, 1200], [S.SpawnerSettings.burst(400, 0.25), S.SpawnerSettings.once(450), S.SpawnerSettings.rate(900.)]),
        (drifting_sparks(1), [4096, 70, 9000], [S.SpawnerSettings.rate(6000.), S.SpawnerSettings.rate(120.), S.SpawnerSettings.burst((500, 1500), (0.1, 0.3))]),
        (ribbon_asset(1), [2500, 6000], [S.SpawnerSettings.rate(3000.), S.SpawnerSettings.burst(2500, 0.5)]),
        (growing_dust(1), [800, 800, 800, 64], [S.SpawnerSettings.rate(400.), S.SpawnerSettings.once(800), S.SpawnerSettings.rate(1000.), S.SpawnerSettings.rate(30.)]),
    ]
    effects, row = [], 0
    for asset, caps, settings in plan:
        effects.append(SceneEffect(ctx, asset, caps, settings, row, dt))
        row += len(caps)
    total_rows = row
    batcher = S.Batcher()
    any_ribbons = any(e.ribbons for e in effects)
    died = 0
    for f in range(90):
        t = np.float32(f) * np.float32(dt)
        # ---- CPU producers: spawner ticks, batching
        batcher.clear()
        spawner_rows, launches_by_batch = [], {}
        for e_idx, e in enumerate(effects):
            counts = [sp.tick(dt) for sp in e.spawners]
            seeds = [int(pcg_hash(np.array([f * 131 + e.first_row + i], dtype=np.uint32))[0]) for i in range(len(counts))]
            e.ref.sim.time = t
            e.ref.set_spawns(counts, seeds)
            for i, inst in enumerate(e.ref.instances):
                g = e.first_row + i
                spawner_rows.append(R.make_spawner(spawn=counts[i], seed=seeds[i], effect_metadata_index=g, draw_indirect_index=g,
                                                   slab_offset=inst.slab_offset))
                key = S.BatchKey(asset_id=e_idx + 1, slab_id=e.slab, pipeline_id=e.effect, property_key=0xFFFFFFFF,
                                 parent_slab_id=0xFFFFFFFF, uses_gpu_events=0, is_cpu_spawner=1)
                b = batcher.push(key, g, inst.slab_offset, counts[i])  # a new batch index, or -1 when merged (batch.rs:348-386)
                if b >= 0:
                    launches_by_batch[b] = e
        infos, prefix, totals = batcher.finish()
        assert len(infos) == len(effects), "instances of one asset in one slab merge into one batch (batch.rs:153-188)"
        # ---- oracle
        for e in effects:
            before = [m.alive_count for m in e.ref.metadata]
            e.oracle.frame(e.ref, orc)
            if any_ribbons and not e.ribbons:
                e.ref.oracle_prefix_sum(orc)  # "hanabi:sort_prefix_sum" runs over EVERY batch when any effect has ribbons
            for i, m in enumerate(e.ref.metadata):
                spawned = min(max(e.ref.spawners[i].spawn, 0), e.ref.instances[i].capacity - before[i])
                died += before[i] + spawned - m.alive_count
        # ---- GPU
        ctx.upload_spawners(spawner_rows)
        ctx.upload_batches(infos, prefix)
        ctx.set_sim_params(dt, float(t), total_rows)
        ctx.simulate([N.BatchLaunch.make(launches_by_batch[b].effect, launches_by_batch[b].slab, b, totals[b]) for b in range(len(infos))])
        # ---- compare every slab and every table row
        ctx.sync()
        gpu_prefix = ctx.read_prefix_sum(0, total_rows)
        for b, e in launches_by_batch.items():
            n = len(e.ref.instances)
            np.testing.assert_array_equal(ctx.slab_download_indirect(e.slab, 0, e.ref.slab_rows), e.ref.indirect, err_msg=f"frame {f} {e.asset.name}: lists")
            np.testing.assert_array_equal(ctx.slab_download_aos(e.slab, 0, e.ref.slab_rows, e.stride), e.ref.particles, err_msg=f"frame {f} {e.asset.name}: particles")
            want_md = e.ref.metadata_rows()
            want_md[:, 5] += e.first_row   # indirect_draw_index is a row of the shared table on the GPU
            got_md = np.stack([np.frombuffer(bytes(ctx.read_metadata(e.first_row + i)), dtype=np.uint32) for i in range(n)])
            np.testing.assert_array_equal(got_md, want_md, err_msg=f"frame {f} {e.asset.name}: metadata")
            assert [ctx.read_draw_args(e.first_row + i).instance_count for i in range(n)] == [int(e.ref.draw[5 * i + 1]) for i in range(n)]
            assert gpu_prefix[e.first_row:e.first_row + n] == e.ref.prefix.tolist()
            bi = ctx.read_batch_info(b)
            assert bi.total_update_count == e.ref.batch_infos[0].total_update_count
            assert [ctx.read_spawner(e.first_row + i).render_pong for i in range(n)] == [e.ref.spawners[i].render_indirect_read_index for i in range(n)]
    assert died > 1000, "the scene must kill and recycle particles"
