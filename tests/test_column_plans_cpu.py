"""Column plans (hnb_effect_column_plan): the pure function from a layout and its HNB_ATTR_UPDATE_READ_ONLY flags to the
slab's columns, the write sets the graph lowering declares, and the generated update on the new plans under the CPU
kernel emulation and in SASS."""
import dataclasses
import os
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from bevy_hanabi_b200 import _native as N
from bevy_hanabi_b200 import graph as G
from bevy_hanabi_b200 import recipes
from bevy_hanabi_b200.runtime import AttrField, LoweredEffect
from tests.effects import firework_trails
from tests.helpers import Instance, RefWorld
from tests.host_exec import HostEffect
from tests.kernel_emu import EmuWorld, assert_same, c5_frame, c5_world

A = G.Attribute
RO = N.ATTR_UPDATE_READ_ONLY
C5_PLAN = [(0, 16), (16, 8), (24, 4), (28, 4)]


def _fx(attrs, stride, flags=0):
    return LoweredEffect("plan", [AttrField(*a) for a in attrs], stride, flags=flags)


def _default_cut(stride):
    out, off = [], 0
    while off < stride:
        w = 16 if stride - off >= 16 else 8 if stride - off >= 8 else 4
        out.append((off, w))
        off += w
    return out


def test_c5_plans():
    assert recipes.c5_asset(64).generate().column_plan() == C5_PLAN
    assert recipes.c5_lowered().column_plan() == [(0, 16), (16, 16)]  # hand-lowered: no write set declared
    lowered = _fx([("position", N.VEC3, 0), ("age", N.FLOAT, 12), ("velocity", N.VEC3, 16), ("lifetime", N.FLOAT, 28, RO)], 32)
    assert lowered.column_plan() == C5_PLAN
    # sector planes and GPU-event emitters keep their cut
    assert dataclasses.replace(lowered, flags=N.EFFECT_SECTOR_PLANES).column_plan() == [(0, 32)]
    assert dataclasses.replace(lowered, flags=N.EFFECT_EMIT_GPU_SPAWN_EVENTS).column_plan() == [(0, 16), (16, 16)]


def test_firework_plan():
    fx = firework_trails(64).generate()
    written = {a.name for a in fx.attrs if not a.flags & RO}
    assert written == {"position", "velocity", "age"}
    plan = fx.column_plan()
    assert plan != _default_cut(fx.particle_stride)
    _check_plan(fx, plan)


def _check_plan(fx, plan):
    """Contiguous, aligned columns, each holding only written or only unwritten words."""
    written = np.zeros(fx.particle_stride // 4, dtype=bool)
    for a in fx.attrs:
        if not a.flags & RO:
            written[a.offset // 4:a.offset // 4 + {N.FLOAT: 1, N.UINT: 1, N.INT: 1, N.VEC2: 2, N.VEC3: 3, N.VEC4: 4}[a.value_type]] = True
    off = 0
    for o, w in plan:
        assert o == off and w in (4, 8, 16) and o % w == 0
        assert len(set(written[o // 4:(o + w) // 4])) == 1, (o, w)
        off += w
    assert off == fx.particle_stride


@pytest.mark.parametrize("stride", [4, 8, 12, 16, 20, 28, 32, 44, 48, 64])
def test_all_written_layout_is_the_default_cut(stride):
    attrs = [(f"f32_{i}", N.FLOAT, 4 * i) for i in range(stride // 4)]
    assert _fx(attrs, stride).column_plan() == _default_cut(stride)


def test_padding():
    # position (written), pad, lifetime (read-only), pad, velocity (written): pads are unwritten words
    fx = _fx([("position", N.VEC3, 0), ("lifetime", N.FLOAT, 16, RO), ("velocity", N.VEC3, 32)], 48)
    assert fx.column_plan() == [(0, 8), (8, 4), (12, 4), (16, 16), (32, 8), (40, 4), (44, 4)]
    _check_plan(fx, fx.column_plan())
    # written words after an unaligned run start on smaller columns until they are aligned
    fx = _fx([("age", N.FLOAT, 0, RO), ("position", N.VEC3, 4), ("velocity", N.VEC4, 16)], 32)
    assert fx.column_plan() == [(0, 4), (4, 4), (8, 8), (16, 16)]
    # padding only, nothing read-only: the default cut, padding stored like today
    fx = _fx([("position", N.VEC3, 0)], 32)
    assert fx.column_plan() == [(0, 16), (16, 16)]


def _update_assets():
    """One asset per update modifier kind; every attribute the update may write is in the layout."""
    c = lambda w: w.lit(G.Vec3(0.5, -1., 2.))
    kinds = {
        "accel": lambda w: [G.AccelModifier(w.lit(G.Vec3(0, -9.8, 0)))],
        "radial": lambda w: [G.RadialAccelModifier(c(w), w.lit(2.5))],
        "tangent": lambda w: [G.TangentAccelModifier(c(w), w.lit(G.Vec3(0, 1, 0)), w.lit(1.5))],
        "conform": lambda w: [G.ConformToSphereModifier(c(w), w.lit(1.5), w.lit(10.), w.lit(5.), w.lit(2.))],
        "drag": lambda w: [G.LinearDragModifier(w.lit(0.7))],
        "kill_sphere": lambda w: [G.KillSphereModifier(c(w), w.lit(4.), False)],
        "kill_aabb": lambda w: [G.KillAabbModifier(c(w), w.lit(G.Vec3(3, 2, 3)), True)],
        "set_attr": lambda w: [G.SetAttributeModifier(A.COLOR, w.attr(A.AGE).vec3(w.lit(0.), w.lit(1.)).vec4_xyz_w(w.lit(1.)).pack4x8unorm())],
        "pos_circle": lambda w: [G.SetPositionCircleModifier(c(w), w.lit(G.Vec3(0, 0, 1)), w.lit(2.), G.VOLUME)],
        "pos_sphere": lambda w: [G.SetPositionSphereModifier(c(w), w.lit(2.), G.SURFACE)],
        "pos_cone": lambda w: [G.SetPositionCone3dModifier(w.lit(3.), w.lit(1.), w.lit(0.2), G.VOLUME)],
        "vel_circle": lambda w: [G.SetVelocityCircleModifier(c(w), w.lit(G.Vec3(0, 0, 1)), w.lit(2.))],
        "vel_sphere": lambda w: [G.SetVelocitySphereModifier(c(w), w.lit(0.3))],
        "vel_tangent": lambda w: [G.SetVelocityTangentModifier(c(w), w.lit(G.Vec3(0, 0, 1)), w.lit(2.))],
        "emit": lambda w: [G.EmitSpawnEventModifier(G.ALWAYS, w.lit(G.U32(1)), 0)],
    }
    out = {}
    for name, update in kinds.items():
        w = G.ExprWriter()
        a = G.EffectAsset(64, w.module, name=name)
        for m in [G.SetAttributeModifier(A.POSITION, w.lit(G.Vec3(0, 0, 0))), G.SetAttributeModifier(A.VELOCITY, w.lit(G.Vec3(0, 1, 0))),
                  G.SetAttributeModifier(A.AGE, w.lit(0.)), G.SetAttributeModifier(A.LIFETIME, w.lit(2.)),
                  G.SetAttributeModifier(A.COLOR, w.lit(G.U32(7))), G.SetAttributeModifier(A.F32_0, w.lit(0.25))]:
            a.init(m)
        for m in update(w):
            a.update(m)
        out[name] = a
    return out


@pytest.mark.parametrize("name", sorted(_update_assets()))
def test_declared_read_only_words_never_change(name):
    """The generated update of every modifier kind, run on random records: no word of an attribute the lowering declared
    read-only changes, and every attribute it declared written may."""
    fx = _update_assets()[name].generate(num_event_bindings=1 if name == "emit" else 0)
    if name == "emit":  # host execution has no event buffers: the declaration alone (an event writes no attribute)
        assert {a.name for a in fx.attrs if not a.flags & RO} == {"position", "age"}
        return
    host = HostEffect(fx)
    rng = np.random.default_rng(7)
    n = 512
    rec = rng.uniform(-3, 3, (n, fx.particle_stride // 4)).astype(np.float32).view(np.uint32)
    before = rec.copy()
    ref = RefWorld(n, fx.particle_stride // 4, [Instance(0, n, alive=n, seed=3)], dt=1 / 30)
    host.update(rec, np.arange(n, dtype=np.uint32), ref.sim, ref.spawners[0])
    ro = [a for a in fx.attrs if a.flags & RO]
    assert {a.name for a in fx.attrs if not a.flags & RO} >= {"position", "age"}
    for a in ro:
        k = {N.VEC3: 3, N.VEC4: 4}.get(a.value_type, 1)
        np.testing.assert_array_equal(rec[:, a.offset // 4:a.offset // 4 + k], before[:, a.offset // 4:a.offset // 4 + k], err_msg=a.name)
    assert "lifetime" in {a.name for a in ro}


class _OnPlan:
    """A lowered effect compiled for a slab of another column plan (what a context compiles on first use)."""

    def __init__(self, fx, plan):
        self._fx, self._plan = fx, plan

    def __getattr__(self, k):
        return getattr(self._fx, k)

    def generate_source(self):
        return self._fx.generate_source_for_plan(self._plan)


def _c5_read_only():
    fx = recipes.c5_lowered()
    return dataclasses.replace(fx, attrs=[dataclasses.replace(a, flags=RO if a.name == "lifetime" else 0) for a in fx.attrs])


@pytest.mark.parametrize("plan", ["own", "default_cut"])
def test_c5_emulated_on_plans(orc, plan):
    """C5 with a read-only lifetime under the emulated kernels, on its own plan and on a default-cut slab: bit-exact
    against the oracle through deaths and spawns into recycled slots."""
    fx = _c5_read_only()
    assert fx.column_plan() == C5_PLAN
    lowered = fx if plan == "own" else _OnPlan(fx, [(0, 16), (16, 16)])
    rng = np.random.default_rng(11)
    ref = c5_world(rng, [Instance(0, 3000, alive=2500, seed=42)])
    emu = EmuWorld(ref, lowered, chunks=2, update_ctas=2)
    for f, spawn in enumerate([0, 400, 0, 300, 0, 0, 250, 0]):
        ref.sim.time = np.float32(f) * ref.sim.delta_time
        c5_frame(orc, ref, emu, spawn)
        assert_same(ref, emu.pull(), f"{plan}: frame {f}")


def _stores(src):
    body = src[src.index("HNB_DI void hnb_store_written"):]
    return re.findall(r"HNB_STORE_PLANE\((\w+), s\.planes\[(\d+)\]", body[:body.index("}")])


def test_update_stores_only_written_columns():
    assert _stores(_c5_read_only().generate_source()) == [("float4", "0"), ("float2", "1"), ("f32", "2")]
    # all-written: the update stores what hnb_store_raw stores
    src = recipes.c5_lowered().generate_source()
    raw = src[src.index("HNB_DI void hnb_store_raw"):]
    assert _stores(src) == re.findall(r"HNB_STORE_PLANE\((\w+), s\.planes\[(\d+)\]", raw[:raw.index("}")]) == [("float4", "0"), ("float4", "1")]
    # on a default-cut slab the read-only effect stores every column holding a written word
    assert _stores(_c5_read_only().generate_source_for_plan([(0, 16), (16, 16)])) == [("float4", "0"), ("float4", "1")]


def _compile(name, src, verbose=False):
    """(ptxas log, SASS of hnb_update) of a generated source, compiled offline for sm_90a with the flags of the NVRTC path."""
    cuda = Path(os.environ.get("CUDA_HOME", "/usr/local/cuda"))
    out = Path(__file__).resolve().parent.parent / "build" / "column_plans"
    out.mkdir(parents=True, exist_ok=True)
    cu, cubin = out / f"{name}.cu", out / f"{name}.cubin"
    cu.write_text(src)
    r = subprocess.run([str(cuda / "bin" / "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--fmad=false",
                        "-diag-suppress", "550,177", "-Xptxas", "-v", "-cubin", str(cu), "-o", str(cubin)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    sass = subprocess.run([str(cuda / "bin" / "cuobjdump"), "-sass", "-fun", "hnb_update", str(cubin)], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def _global_stores(sass):
    return re.findall(r"STG\.E(\.128|\.64|)\s", sass)


def test_c5_update_sass():
    """sm_90a SASS of the C5 update on its plan: per row in flight (four), one 128-, one 64- and one 32-bit store (columns
    0-2) where the all-written C5 has two 128-bit stores, and no store of the lifetime column; at most 80 registers (3 CTAs
    of 256 threads per SM) and no spills."""
    log, sass = _compile("c5_plan", _c5_read_only().generate_source())
    update = log[log.index("hnb_update"):]
    regs = int(re.search(r"Used (\d+) registers", update).group(1))
    assert regs <= 80 and "0 bytes spill stores" in update, update[:400]
    _, sass_all = _compile("c5_all_written", recipes.c5_lowered().generate_source())
    got, base = _global_stores(sass), _global_stores(sass_all)
    assert got.count(".128") == 4 and base.count(".128") == 8
    assert got.count(".64") == base.count(".64") + 4
    assert got.count("") == base.count("") + 4, "exactly one 32-bit store per row: column 2, not the lifetime column"


def test_all_written_update_sass_is_the_store_raw_update():
    """An all-written effect: hnb_update calling hnb_store_written compiles to the same SASS as calling hnb_store_raw (what
    the update called before column plans)."""
    src = recipes.c5_lowered().generate_source()
    call = "hnb_store_written(raw[k], P.slab, base_particle + pidx[k]);"
    assert src.count(call) == 1
    _, a = _compile("c5_written_call", src)
    _, b = _compile("c5_raw_call", src.replace(call, "hnb_store_raw(raw[k], P.slab, base_particle + pidx[k]);"))
    strip = lambda t: [l for l in t.splitlines() if "Function" not in l and ".cubin" not in l and "code for" not in l]
    assert strip(a) == strip(b)
