"""The drawn assets of tests/plan_assets.py reach every plan shape the record kernels branch on (DESIGN.md §3), read from
`column_plan()` and `hnb_effect_column_words` with no GPU. This keeps the generator, and so tests/test_gpu_plan_shapes.py,
from quietly becoming narrow when the planner changes."""
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import graph as G
from tests.effects import tile_k
from tests.plan_assets import SEEDS, default_cut, draw, is_word_map


def _runs(stride, attrs):
    """Columns of the runs plan: every maximal run of written and of unwritten words cut into aligned 16-, 8- and 4-byte
    columns (restated from DESIGN.md §3)."""
    written = [False] * (stride // 4)
    for a in attrs:
        if not a.flags & N.ATTR_UPDATE_READ_ONLY:
            for c in range(G.vt_count(a.value_type)):
                written[a.offset // 4 + c] = True
    n, w = 0, 0
    while w < len(written):
        end = w
        while end < len(written) and written[end] == written[w]:
            end += 1
        off = 4 * w
        while off < 4 * end:
            width = 16
            while width > 4 and (off % width or off + width > 4 * end):
                width //= 2
            n, off = n + 1, off + width
        w = end
    return n


@pytest.fixture(scope="module")
def shapes():
    """Per shape, the seeds whose plan has it."""
    out = {}

    def has(shape, seed):
        out.setdefault(shape, set()).add(seed)

    for seed in SEEDS:
        d = draw(seed)
        fx = d.asset.generate()
        plan, words, stride = fx.column_plan(), fx.column_words(), fx.particle_stride
        off = {a.name: a.offset // 4 for a in fx.attrs}
        mapped = is_word_map(words)
        assert [w for _, w in plan] == [4 * len(ws) for ws in words]
        assert sorted(x for ws in words for x in ws) == list(range(stride // 4)), f"seed {seed}: every word in one column"
        has(("stride", stride), seed)
        has(("K", tile_k(stride)), seed)
        has("word map" if mapped else "default cut" if plan == default_cut(stride) else "runs", seed)
        for (o, width), ws in zip(plan, words):
            if 4 * ws[0] % 16:
                has(("column at a record offset off 16 bytes", width), seed)
            if width == 8 and ws[0] % 2:
                has("8-byte column at an odd word", seed)
            if mapped and ws != list(range(ws[0], ws[0] + len(ws))):
                has(("word-map column of words not consecutive", len(ws)), seed)
            if mapped and len(ws) == 1 and 4 * ws[0] != o:
                has(("word-map column of words not consecutive", 1), seed)
        p = off["position"]
        cols = {i for i, ws in enumerate(words) for x in ws if p <= x < p + 3}
        if len(cols) > 1:
            has("position split" + (" in a word map" if mapped else ""), seed)
        elif len(words[cols.pop()]) == 4:
            has("position in one 16-byte column", seed)
        if mapped:
            assert off["age"] < off["lifetime"], "the reference's layout sorts scalars by name: age comes first"
            life = words.index([off["lifetime"]])
            has("lifetime in the last column" if life == len(words) - 1 else "lifetime before another column", seed)
            assert words[life - 1] == [off["age"]], "the age column comes right before the lifetime column"
        if len(plan) == 16:
            has("16 columns", seed)
        if _runs(stride, fx.attrs) > 16:
            assert plan == default_cut(stride)
            has("more than 16 runs: the default cut", seed)
        if "ribbon_id" in off:
            has("ribbon" + (" in a word map" if mapped else ""), seed)
    return out


SHAPES = ([("column at a record offset off 16 bytes", w) for w in (4, 8, 16)] + ["8-byte column at an odd word"]
          + [("word-map column of words not consecutive", n) for n in (1, 2, 4)]
          + ["lifetime in the last column", "lifetime before another column", "position in one 16-byte column", "position split",
             "position split in a word map",             "16 columns", "more than 16 runs: the default cut", "word map", "runs", "default cut", "ribbon",
             "ribbon in a word map", ("K", 1), ("K", 2), ("K", 4)])


@pytest.mark.parametrize("shape", SHAPES, ids=str)
def test_drawn_set_reaches(shapes, shape):
    assert shapes.get(shape), f"no drawn asset has {shape}"


def test_strides_span_the_range(shapes):
    """From the smallest record that holds a position (16 bytes: position and age) to 256 bytes (16 default-cut columns)."""
    strides = sorted(s for k, s in [k for k in shapes if isinstance(k, tuple) and k[0] == "stride"])
    assert strides[0] <= 32 and strides[-1] == 256 and len(strides) >= 10, strides


def test_draw_is_deterministic():
    for seed in SEEDS[:6]:
        a, b = draw(seed).asset.generate(), draw(seed).asset.generate()
        assert (a.attrs, a.init_code, a.update_code) == (b.attrs, b.init_code, b.update_code)


def test_word_maps_come_from_read_only_lifetimes():
    """Even seeds keep the lifetime read-only and reap-only; only they may give word maps."""
    for seed in SEEDS:
        d = draw(seed)
        fx = d.asset.generate()
        if is_word_map(fx.column_words()):
            assert d.word_map_wanted and "lifetime" not in d.written, f"seed {seed}"
