"""The fast oracle of the churned full-size tests (tests/test_gpu_churn_fullsize.py) against the authority it stands in for.

At 16 Mi slots the numpy interpreter (oracle.hanabi_oracle.EffectOracle) takes seconds per frame, so those tests step
drifting_sparks with C bodies: orc_body_init_sparks for the init and orc_body_update_c5 with ACCEL_DRAG for the update,
the update run by orc_update_c5_parallel, and slot order read through lists sorted by a presence mask. Here each of these
equals what it replaces, bit for bit, on churned 4096-slot worlds whose dead stacks are shuffled and whose alive lists are
permutations of the slab."""
import numpy as np
import pytest

from oracle.hanabi_oracle import EffectOracle
from tests.effects import ACCEL_DRAG, sparks_init
from tests.helpers import sorted_slots, sparks_world

DT = 1.0 / 60.0


def c_frame(ref, orc, f, spawns, init_user):
    """Frame f of a drifting_sparks world under the C bodies (the GPU tests' oracle)."""
    ref.sim.time = ref.sim.virtual_time = ref.sim.real_time = np.float32(f) * ref.sim.delta_time
    ref.set_spawns(spawns, [1000 + 7 * i + f for i in range(len(spawns))])
    ref.oracle_frame(orc, orc.orc_body_update_c5(), ACCEL_DRAG, orc.orc_body_init_sparks(), init_user)


def np_frame(ref, orc, eo, f, spawns):
    ref.sim.time = ref.sim.virtual_time = ref.sim.real_time = np.float32(f) * ref.sim.delta_time
    ref.set_spawns(spawns, [1000 + 7 * i + f for i in range(len(spawns))])
    eo.frame(ref, orc)


def assert_same(a, b, what):
    np.testing.assert_array_equal(a.particles, b.particles, err_msg=f"{what}: records")
    np.testing.assert_array_equal(a.indirect, b.indirect, err_msg=f"{what}: lists and dead stack")
    np.testing.assert_array_equal(a.metadata_rows(), b.metadata_rows(), err_msg=f"{what}: metadata")
    np.testing.assert_array_equal(a.draw, b.draw, err_msg=f"{what}: draw args")


def permuted(ref, i=0):
    """Whether instance i's alive list is far from sorted (a churned gather, not a run of slots)."""
    md, base = ref.metadata[i], ref.instances[i].slab_offset
    lst = ref.indirect[base:base + md.alive_count, md.indirect_write_index].astype(np.int64)
    return len(lst) > 64 and np.median(np.abs(np.diff(lst))) > 16


@pytest.mark.parametrize("slot", [False, True], ids=["list", "slot"])
@pytest.mark.parametrize("lifetime,rate", [((0.2, 0.9), 4096 // 40), ((0.05, 0.3), 4096 // 12)], ids=["0.2-0.9", "0.05-0.3"])
def test_c_bodies_equal_numpy_oracle(orc, lifetime, rate, slot):
    """orc_body_init_sparks + orc_body_update_c5 equal EffectOracle after each of 60 frames of churn (spawns into a shuffled
    dead stack, deaths every frame), in list order and in slot order."""
    from tests.effects import drifting_sparks
    asset = drifting_sparks(4096, lifetime=lifetime)
    _, ref_np = sparks_world([4096], dt=DT)
    _, ref_c = sparks_world([4096], dt=DT)
    assert not (ref_np.indirect[:, 2] == np.arange(4096)).all(), "the dead stack must be shuffled"
    ref_np.slot_order = ref_c.slot_order = slot
    eo, user = EffectOracle(asset), sparks_init(lifetime)
    for f in range(60):
        np_frame(ref_np, orc, eo, f, [rate])
        c_frame(ref_c, orc, f, [rate], user)
        assert_same(ref_c, ref_np, f"frame {f}")
    md = ref_c.metadata[0]
    assert 0 < md.alive_count < 4096 and md.particle_counter > 4096, "the world must churn: spawns recycle dead slots"
    assert slot or permuted(ref_c)  # slot order writes its survivors in slot order


def churned_pair(orc, caps, threads, slot, frames=48):
    """Two copies of a drifting_sparks world of instances `caps` in one batch, stepped under the C bodies, one with the
    serial orc_update and one with orc_update_c5_parallel on `threads` threads; compared after every frame."""
    _, serial = sparks_world(caps, dt=DT)
    _, par = sparks_world(caps, dt=DT)
    serial.slot_order = par.slot_order = slot
    par.parallel_c5 = threads
    user = sparks_init()
    rates = [c // 30 for c in caps]
    for f in range(frames):
        c_frame(serial, orc, f, rates, user)
        c_frame(par, orc, f, rates, user)
        assert_same(par, serial, f"{threads} threads, frame {f}")
    return par


@pytest.mark.parametrize("slot", [False, True], ids=["list", "slot"])
@pytest.mark.parametrize("threads", [1, 3, "max"])
def test_parallel_update_equals_serial(orc, threads, slot):
    n = orc.orc_max_threads() if threads == "max" else threads
    ref = churned_pair(orc, [4096], n, slot)
    assert slot or permuted(ref)


@pytest.mark.parametrize("threads", [1, 3, "max"])
def test_parallel_update_two_instance_batch(orc, threads):
    """One batch of two instances (capacities not multiples of 32): the parallel update runs per instance, in batch order."""
    n = orc.orc_max_threads() if threads == "max" else threads
    ref = churned_pair(orc, [2500, 1700], n, False)
    assert ref.batches == [[0, 1]]
    assert all(0 < ref.metadata[i].alive_count < c for i, c in enumerate([2500, 1700]))
    assert permuted(ref, 0) and permuted(ref, 1)


def test_sorted_slots_equals_np_sort(orc):
    """The presence-mask sort of slot order equals np.sort on churned lists, and falls back to np.sort on a list that is
    not a set of distinct slots of the slice."""
    _, ref = sparks_world([4096], dt=DT)
    user = sparks_init()
    seen = 0
    for f in range(40):
        c_frame(ref, orc, f, [4096 // 40], user)
        md = ref.metadata[0]
        for col in (0, 1):
            lst = ref.indirect[:md.alive_count, col]
            np.testing.assert_array_equal(sorted_slots(lst, 4096), np.sort(lst))
        seen += permuted(ref)
    assert seen > 20
    for odd in ([], [5, 5, 1], [4096, 3], [7, 0, 4095]):
        lst = np.array(odd, dtype=np.uint32)
        got = sorted_slots(lst, 4096)
        assert got.dtype == np.uint32 or len(lst) == 0
        np.testing.assert_array_equal(got, np.sort(lst))
