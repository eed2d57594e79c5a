"""Drawn graph assets for the layout layer: a seeded, deterministic generator of `graph.EffectAsset`s whose layouts reach
the column plans DESIGN.md §3 describes (runs plans, word maps, the default-cut fallback), so that every reader and writer
of slab records can be held to the oracle's AoS bytes on plans no hand-written effect has.

Every expression is exact in IEEE fp32 without contraction (literals, rand scaled by powers of two, add, mul, Accel,
LinearDrag), so the numpy interpreter equals the device bit for bit. Even seeds keep `lifetime` read-only and reap-only
beside an f32 `age`, which gives word maps where the plan allows one; odd seeds write the lifetime or leave it out, which
gives runs plans. Test infrastructure only."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from bevy_hanabi_b200 import graph as G

A = G.Attribute

F32 = ["alpha", "size", "f32_0", "f32_1", "f32_2", "f32_3"]
U32 = ["color", "u32_0", "u32_1", "u32_2", "u32_3"]
VEC2 = ["size2", "f32x2_0", "f32x2_1", "f32x2_2", "f32x2_3"]
VEC3 = ["size3", "axis_x", "axis_y", "axis_z", "f32x3_0", "f32x3_1", "f32x3_2", "f32x3_3"]
VEC4 = ["hdr_color", "f32x4_0", "f32x4_1", "f32x4_2", "f32x4_3"]
CAPACITY = 4096
DT = 0.05
MAX_STRIDE = 256

# The drawn set: the first 40 seeds, then seeds that reach a shape none of those does (tests/test_plan_shapes_cpu.py):
# 54 and 81 give word-map columns of two words that are not consecutive.
SEEDS = list(range(40)) + [54, 81]


@dataclass
class Drawn:
    seed: int
    asset: G.EffectAsset
    names: list[str]          # the attributes of the layout
    written: set[str]         # attributes the update writes (age code, Euler integration and modifiers included)
    word_map_wanted: bool     # lifetime read-only and reap-only beside an f32 age


def _pow2(rng, lo, hi):
    return float(2.0 ** int(rng.integers(lo, hi + 1)))


def _init_value(w, rng, name, vt):
    n, elem = G.vt_count(vt), G.vt_elem(vt)
    if name == "ribbon_id":
        return (w.rand(G.FLOAT) * w.lit(4.)).cast(G.UINT)
    if elem == "u":
        return (w.rand(G.FLOAT) * w.lit(1024.)).cast(G.UINT) if rng.random() < 0.5 else w.lit(G.U32(int(rng.integers(0, 2**32))))
    r = w.rand(G.FLOAT) if n == 1 else w.rand(G.vt_make("f", n))
    return r * w.lit(_pow2(rng, -1, 3)) - w.lit(_pow2(rng, -2, 1))


def _update_value(w, rng, name, vt):
    if G.vt_elem(vt) == "u":
        return w.attr(A.by_name(name)) + w.lit(G.U32(int(rng.integers(1, 2**31))))
    return w.attr(A.by_name(name)) * w.lit(1. - _pow2(rng, -6, -3)) + w.lit(_pow2(rng, -8, -4))


def _stride(names):
    try:
        return G.particle_layout_of(names)[1]
    except G.HanabiError:  # more padding fields than a layout may have: far above MAX_STRIDE
        return MAX_STRIDE + 1


def draw(seed: int) -> Drawn:
    """The asset of `seed`: deterministic across runs and machines (numpy's PCG64 stream of the seed)."""
    rng = np.random.default_rng([0x91A5, seed])
    word_map = seed % 2 == 0
    size = rng.choice(["tiny", "small", "medium", "large"], p=[0.15, 0.35, 0.3, 0.2])
    budget = {"tiny": 0, "small": 4, "medium": 10, "large": 24}[size]
    pool = F32 + U32 + VEC2 + VEC3 + VEC4
    extra = list(rng.choice(pool, size=min(budget + int(rng.integers(0, 4)), len(pool)), replace=False)) if budget else []
    if size == "tiny":
        extra = list(rng.choice(F32 + U32, size=int(rng.integers(0, 2)), replace=False))
    names = ["age", "position"]  # every asset needs a position
    if word_map or rng.random() < 0.7:
        names.append("lifetime")
    if rng.random() < 0.5:
        names.append("velocity")
    if rng.random() < 0.3:
        names.append("ribbon_id")
    names += [str(n) for n in extra]
    while _stride(names) > MAX_STRIDE:  # 16 default-cut columns at most
        names.pop()

    w = G.ExprWriter()
    asset = G.EffectAsset(CAPACITY, w.module, name=f"drawn_{seed}")
    if rng.random() < 0.25:
        asset.with_motion_integration(G.MOTION_NONE)
    written = {"age"}
    for name in names:
        vt = A.by_name(name).vt
        if name == "age":
            value = w.lit(0.) if rng.random() < 0.7 else w.rand(G.FLOAT) * w.lit(0.125)
        elif name == "lifetime":
            value = w.lit(0.15).uniform(w.lit(0.6))
        else:
            value = _init_value(w, rng, name, vt)
        asset.init(G.SetAttributeModifier(A.by_name(name), value))
    if "velocity" in names:
        if rng.random() < 0.6:
            asset.update(G.AccelModifier(w.lit(G.Vec3(0., -_pow2(rng, 0, 3), _pow2(rng, -2, 0)))))
            written.add("velocity")
        if rng.random() < 0.5:
            asset.update(G.LinearDragModifier(w.lit(_pow2(rng, -2, 1))))
            written.add("velocity")
        if "position" in names and asset.motion_integration != G.MOTION_NONE:
            written.add("position")
    if "lifetime" in names and not word_map:
        asset.update(G.SetAttributeModifier(A.LIFETIME, w.attr(A.LIFETIME) + w.lit(0.0078125)))
        written.add("lifetime")
    for name in names:
        if name in ("age", "lifetime", "ribbon_id", "velocity") or (name == "position" and name in written):
            continue
        if rng.random() < 0.5:
            asset.update(G.SetAttributeModifier(A.by_name(name), _update_value(w, rng, name, A.by_name(name).vt)))
            written.add(name)
    return Drawn(seed, asset, names, written, word_map)


def is_word_map(words) -> bool:
    """Whether a plan's column words (hnb_effect_column_words) hold a column whose words are not consecutive."""
    return any(ws != list(range(ws[0], ws[0] + len(ws))) for ws in words)


def default_cut(stride: int) -> list[tuple[int, int]]:
    out, off = [], 0
    while off < stride:
        w = 16 if stride - off >= 16 else 8 if stride - off >= 8 else 4
        out.append((off, w))
        off += w
    return out
