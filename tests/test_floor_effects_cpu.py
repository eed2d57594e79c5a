"""Which effects keep lifetime floors (DESIGN.md §3): every effect of tests/effects.py and bevy_hanabi_b200/recipes.py with
its column plan, whether its module is generated with HNB_LIFE_FLOOR 1, and its K (rows in flight per lane). An effect
keeps floors when its lifetime is a reap-only f32 in a 4-byte column of its own; it uses them once a fill, a repack or a
restore gives an instance its identity claim. The effects listed with floors at K = 2 and K = 1 run on the device in
tests/test_gpu_floor_shapes.py, C5 at every K there too."""
import pytest

from bevy_hanabi_b200 import recipes
from tests import effects as E

C5_PLAN = [(0, 16), (16, 8), (24, 4), (28, 4)]
DEFAULT_32 = [(0, 16), (16, 16)]
DEFAULT_48 = [(0, 16), (16, 16), (32, 16)]
WIDE_144 = [(16 * i, 16) for i in range(9)]

# name -> (module, column plan, HNB_LIFE_FLOOR 1, K)
EXPECTED = {
    "c5_asset": (lambda: recipes.c5_asset(4096).generate(), C5_PLAN, True, 4),
    "c5_lowered": (lambda: recipes.c5_lowered(), DEFAULT_32, False, 4),
    "firework_trails": (lambda: E.firework_trails(4096).generate(), [(0, 16), (16, 8), (24, 4), (28, 4), (32, 16)], False, 2),
    "force_field": (lambda: E.force_field(4096).generate(), C5_PLAN, True, 4),
    "drifting_sparks": (lambda: E.drifting_sparks(4096).generate(), C5_PLAN, True, 4),
    "growing_dust": (lambda: E.growing_dust(4096).generate(), DEFAULT_32, False, 4),
    "ribbon_asset": (lambda: E.ribbon_asset(4096).generate(), DEFAULT_48, False, 2),
    "instancing": (lambda: E.instancing(4096).generate(), DEFAULT_32, False, 4),
    "matrix_asset": (lambda: E.matrix_asset(4096).generate(), WIDE_144, False, 1),
    "vec4x2_64": (lambda: E.table_asset("vec4x2_64", 4096).generate(), [(0, 16), (16, 16), (32, 16), (48, 8), (56, 4), (60, 4)], True, 2),
    "vec4x4_96": (lambda: E.table_asset("vec4x4_96", 4096).generate(),
                  [(0, 16), (16, 16), (32, 16), (48, 16), (64, 16), (80, 8), (88, 4), (92, 4)], True, 1),
    # effects that emit GPU spawn events keep the default cut, where the lifetime shares a column with the velocity
    "event_assets.parent": (lambda: E.event_assets()[0].generate(num_event_bindings=1), DEFAULT_32, False, 4),
    "event_assets.child": (lambda: E.event_assets()[1].generate(parent=E.event_assets()[0]), DEFAULT_48, False, 2),
    "emitter_assets.parent": (lambda: E.emitter_assets(4096)[0].generate(num_event_bindings=2), DEFAULT_32, False, 4),
    "emitter_assets.child": (lambda: E.emitter_assets(4096)[1][0].generate(parent=E.emitter_assets(4096)[0]), DEFAULT_48, False, 2),
}


@pytest.fixture(autouse=True)
def _default_shape(monkeypatch):
    for v in ("HNB_TILE_K", "HNB_ROWS_PER_LANE", "HNB_DEFINES"):
        monkeypatch.delenv(v, raising=False)


@pytest.mark.parametrize("name", list(EXPECTED))
def test_column_plan_floors_and_k(name):
    build, plan, floors, k = EXPECTED[name]
    fx = build()
    src = fx.generate_source()
    got = (fx.column_plan(), "\n#define HNB_LIFE_FLOOR 1\n" in src, f"\n#define HNB_TILE_K {k}\n" in src)
    print(f"{name}: {fx.particle_stride} B, plan {got[0]}, floors {got[1]}, K {k}")
    assert got == (plan, floors, True)
    assert E.tile_k(fx.particle_stride) == k


def test_every_effect_is_listed():
    """A builder added to tests/effects.py or recipes.py must be entered above."""
    import inspect
    builders = {n for n, f in inspect.getmembers(E, inspect.isfunction) if f.__module__ == E.__name__ and not n.startswith("_")}
    builders -= {"table_asset", "table_props", "tile_k", "edge_counts", "c5_init", "fill_c5", "exact_expr"}  # not effects
    listed = {n.split(".")[0] for n in EXPECTED}
    assert builders <= listed, f"not listed: {sorted(builders - listed)}"
    assert set(E.EFFECTS) - {"trails48", "matrix144"} <= listed  # trails48 and matrix144 are firework_trails and matrix_asset
    recipe_fns = {n for n, f in inspect.getmembers(recipes, inspect.isfunction) if f.__module__ == recipes.__name__}
    assert recipe_fns - {"c5_generated_source"} <= listed, f"not listed: {sorted(recipe_fns - listed)}"
