"""The sector-plane slab layout on the device."""
import numpy as np
import pytest

from oracle.hanabi_oracle import pcg_hash
from tests.effects import drifting_sparks, firework_trails, ribbon_asset
from tests.helpers import Instance, Lockstep, RefWorld

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["sparks", "trails", "ribbons"])
def test_sector_planes_on_the_device(ctx, orc, name):
    """HNB_SLAB_SECTOR_PLANES + HNB_EFFECT_SECTOR_PLANES: same results as the default layout (32-, 48-byte records, and a
    ribbon effect through the sort's key gathers), including AoS upload / download of the interleaved columns."""
    asset = {"sparks": drifting_sparks, "trails": firework_trails, "ribbons": ribbon_asset}[name](6000)
    fields, size, _ = asset.particle_layout()
    ref = RefWorld(6000, size // 4, [Instance(0, 6000, alive=0, seed=4)], dt=1 / 10)
    if name == "ribbons":
        ref.set_sort_keys(fields)
    seeds = lambda n, f: [int(pcg_hash(np.array([f + 300], dtype=np.uint32))[0])]
    Lockstep(ctx, orc, ref, asset, sector=True, seeds=seeds).run([[2500 if f % 3 == 0 else 120] for f in range(8)], what=name)
