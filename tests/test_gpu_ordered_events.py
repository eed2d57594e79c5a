"""HNB_EFFECT_ORDERED_EVENTS on the device."""
import pytest

from tests.helpers import at_tile_sizes, emitter_scene, tiled_ctx  # noqa: F401

pytestmark = pytest.mark.gpu


@at_tile_sizes("pcap", [1024, 6000])
def test_ordered_events_two_children(tiled_ctx, orc, pcap):
    """HNB_EFFECT_ORDERED_EVENTS on the device : with
    ordered append the buffers must hold EXACTLY the canonical sequence, overflow included, and the children need no
    re-ordering of the oracle's events. With the slab-size rule and at 2-4 forced sub-tiles per tile: an event's row is row0 + (j*K + k)*32 + lane. Scenario: one parent, two event channels: channel 0 fed every frame by particles that are alive (EventEmitCondition::Always,
    count 0 or 1 drawn per particle), channel 1 by dying particles (OnDie, 4 events each). Each child consumes its
    own buffer the frame after. Children come BEFORE the parent in batch order, as EffectSorter places them
    (batch.rs:599-603), so a child's init reads the parent's records before the parent's init recycles slots."""
    tiled_ctx.tile_batch = 2  # the parent: 32-byte records, 128-row sub-tiles (the children's 48-byte records have 64-row ones)
    emitter_scene(tiled_ctx, orc, pcap, ordered=True)
