"""Authoring API: Python mirror of the reference's ``Module`` / ``ExprWriter`` / ``WriterExpr`` /
modifiers / ``EffectAsset`` (src/graph/expr.rs, src/modifier/*.rs, src/asset.rs), implemented as a
binding over the Level-2 C ABI (``include/hanabi_b200_graph.h``). All lowering (expression -> CUDA C,
layouts, code generation) happens in the native library; this module only forwards calls and keeps a
light record of the graph (``Module.nodes``, ``EffectAsset.init_modifiers`` ...) that the test oracle
walks to interpret the same effect independently.
"""
from __future__ import annotations

import ctypes as C
import struct
from dataclasses import dataclass, field
from typing import Optional, Sequence, Union

from . import _native as N
from ._native import HanabiError, check, lib
from .runtime import AttrField, LoweredEffect

P = C.POINTER
u32 = C.c_uint32

_SIGS = {
    "hnb_module_create": (C.c_void_p, []),
    "hnb_module_destroy": (None, [C.c_void_p]),
    "hnb_module_lit": (u32, [C.c_void_p, u32, P(u32)]),
    "hnb_module_attr": (u32, [C.c_void_p, C.c_char_p]),
    "hnb_module_parent_attr": (u32, [C.c_void_p, C.c_char_p]),
    "hnb_module_add_property": (u32, [C.c_void_p, C.c_char_p, u32, P(u32)]),
    "hnb_module_prop": (u32, [C.c_void_p, u32]),
    "hnb_module_builtin": (u32, [C.c_void_p, u32, u32]),
    "hnb_module_unary": (u32, [C.c_void_p, u32, u32]),
    "hnb_module_binary": (u32, [C.c_void_p, u32, u32, u32]),
    "hnb_module_ternary": (u32, [C.c_void_p, u32, u32, u32, u32]),
    "hnb_module_cast": (u32, [C.c_void_p, u32, u32]),
    "hnb_module_is_const": (C.c_int32, [C.c_void_p, u32]),
    "hnb_module_has_side_effect": (C.c_int32, [C.c_void_p, u32]),
    "hnb_module_eval": (C.c_int32, [C.c_void_p, u32, u32, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]),
    "hnb_attribute_count": (u32, []),
    "hnb_attribute_info": (C.c_int32, [u32, P(C.c_char_p), P(u32), P(u32)]),
    "hnb_particle_layout_build": (C.c_int32, [P(C.c_char_p), u32, P(N.AttrLayout), u32, P(u32), P(u32), P(u32)]),
    "hnb_format_f32": (C.c_int32, [C.c_float, C.c_char_p, C.c_size_t]),
    "hnb_asset_create": (C.c_void_p, [C.c_char_p, u32, C.c_void_p]),
    "hnb_asset_destroy": (None, [C.c_void_p]),
    "hnb_asset_set_simulation_space": (C.c_int32, [C.c_void_p, u32]),
    "hnb_asset_set_motion_integration": (C.c_int32, [C.c_void_p, u32]),
    "hnb_asset_add_modifier": (C.c_int32, [C.c_void_p, u32, u32, P(u32), u32, P(u32), u32]),
    "hnb_asset_particle_layout": (C.c_int32, [C.c_void_p, P(N.AttrLayout), u32, P(u32), P(u32), P(u32)]),
    "hnb_asset_property_layout": (C.c_int32, [C.c_void_p, P(N.AttrLayout), u32, P(u32), P(u32)]),
    "hnb_asset_serialize_properties": (C.c_int32, [C.c_void_p, P(C.c_char_p), P(P(u32)), u32, C.c_void_p, u32, P(u32)]),
    "hnb_module_len": (u32, [C.c_void_p]),
    "hnb_module_get": (C.c_int32, [C.c_void_p, u32, C.c_void_p]),
    "hnb_node_graph_create": (C.c_void_p, []),
    "hnb_node_graph_destroy": (None, [C.c_void_p]),
    "hnb_node_graph_add_node": (u32, [C.c_void_p, u32, C.c_char_p]),
    "hnb_node_graph_node_count": (u32, [C.c_void_p]),
    "hnb_node_graph_link": (C.c_int32, [C.c_void_p, u32, u32]),
    "hnb_node_graph_unlink": (C.c_int32, [C.c_void_p, u32, u32]),
    "hnb_node_graph_unlink_all": (C.c_int32, [C.c_void_p, u32]),
    "hnb_node_graph_slots": (C.c_int32, [C.c_void_p, u32, u32, P(u32), u32, P(u32)]),
    "hnb_node_graph_find_slot": (u32, [C.c_void_p, u32, u32, C.c_char_p]),
    "hnb_node_graph_slot_info": (C.c_int32, [C.c_void_p, u32, P(C.c_char_p), P(u32), P(u32), P(C.c_int32), P(u32), u32, P(u32)]),
    "hnb_node_graph_eval_node": (C.c_int32, [C.c_void_p, u32, C.c_void_p, P(u32), u32, P(u32), u32, P(u32)]),
    "hnb_node_graph_eval_slot": (C.c_int32, [C.c_void_p, C.c_void_p, u32, P(u32)]),
    "hnb_effect_properties_create": (C.c_void_p, []),
    "hnb_effect_properties_destroy": (None, [C.c_void_p]),
    "hnb_effect_properties_len": (u32, [C.c_void_p]),
    "hnb_effect_properties_set": (C.c_int32, [C.c_void_p, C.c_char_p, u32, P(u32)]),
    "hnb_effect_properties_set_if_changed": (C.c_int32, [C.c_void_p, C.c_char_p, u32, P(u32), P(u32)]),
    "hnb_effect_properties_get_stored": (C.c_int32, [C.c_void_p, C.c_char_p, P(u32), P(u32)]),
    "hnb_effect_properties_get": (C.c_int32, [C.c_void_p, u32, P(C.c_char_p), P(u32), P(u32), P(u32)]),
    "hnb_effect_properties_update": (C.c_int32, [C.c_void_p, C.c_void_p, P(u32)]),
    "hnb_effect_properties_serialize": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, u32, P(u32)]),
    "hnb_asset_generate": (C.c_int32, [C.c_void_p, C.c_void_p, u32, P(C.c_void_p)]),
    "hnb_generated_desc": (C.c_int32, [C.c_void_p, P(N.EffectDesc)]),
    "hnb_generated_destroy": (None, [C.c_void_p]),
}
for _n, (_r, _a) in _SIGS.items():
    _f = getattr(lib, _n)
    _f.restype = _r
    _f.argtypes = _a
GRAPH_SIGNATURES = _SIGS

# ---------------------------------------------------------------------------------------------------
# Value types and values
# ---------------------------------------------------------------------------------------------------
BOOL, FLOAT, INT, UINT = N.BOOL, N.FLOAT, N.INT, N.UINT
VEC2, VEC3, VEC4 = N.VEC2, N.VEC3, N.VEC4
_ELEM = {0: "b", 1: "f", 2: "i", 3: "u"}


# matCxR<f32> codes (hnb_value_type): (columns, rows)
_MAT_DIMS = {16: (2, 2), 17: (3, 3), 18: (4, 4), 19: (2, 3), 20: (2, 4), 21: (3, 2), 22: (3, 4), 23: (4, 2), 24: (4, 3)}
MAT2, MAT3, MAT4 = 16, 17, 18


def vt_is_matrix(vt: int) -> bool:
    return vt >= 16


def vt_matrix_dims(vt: int) -> tuple:
    """(columns, rows) of a matrix type."""
    return _MAT_DIMS[vt]


def vt_matrix(cols: int, rows: int) -> int:
    """MatrixType::new(cols, rows) (reference src/attributes.rs:358-362)."""
    for vt, d in _MAT_DIMS.items():
        if d == (cols, rows):
            return vt
    raise ValueError("matrix sizes are 2..4 columns by 2..4 rows")


def vt_count(vt: int) -> int:
    """Number of 32-bit lanes of a value (matrix: columns x rows, stored column by column)."""
    if vt >= 16:
        c, r = _MAT_DIMS[vt]
        return c * r
    return 1 if vt < 4 else 2 + (vt - 4) % 3


def vt_elem(vt: int) -> str:
    """'b', 'f', 'i' or 'u'"""
    if vt < 4:
        return _ELEM[vt]
    if vt >= 16:
        return "f"
    return "bfiu"[(vt - 4) // 3]


def vt_make(elem: str, count: int) -> int:
    base = "bfiu".index(elem)
    return base if count == 1 else 4 + 3 * base + (count - 2)


def _f32_bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


@dataclass(frozen=True)
class Value:
    """A typed constant: ``vt`` is an hnb_value_type, ``words`` its 32-bit lanes."""
    vt: int
    words: tuple

    @staticmethod
    def of(x) -> "Value":
        if isinstance(x, Value):
            return x
        if isinstance(x, bool):
            return Value(BOOL, (0xFFFFFFFF if x else 0,))
        if isinstance(x, float):
            return Value(FLOAT, (_f32_bits(x),))
        if isinstance(x, int):
            raise TypeError("integer literals are ambiguous: use U32(x) or I32(x)")
        if isinstance(x, (tuple, list)):
            if all(isinstance(c, bool) for c in x):
                return Value(vt_make("b", len(x)), tuple(0xFFFFFFFF if c else 0 for c in x))
            if all(isinstance(c, (float, int)) and not isinstance(c, bool) for c in x):
                return Value(vt_make("f", len(x)), tuple(_f32_bits(float(c)) for c in x))
        raise TypeError(f"cannot make a literal from {x!r}")

    def floats(self):
        return [struct.unpack("<f", struct.pack("<I", w))[0] for w in self.words]

    @staticmethod
    def splat(scalar, count: int) -> "Value":
        """VectorValue::splat (graph/mod.rs:572-590): a vector of `count` copies of a scalar value."""
        v = Value.of(scalar)
        if v.vt not in (BOOL, FLOAT, INT, UINT) or not 2 <= count <= 4:
            raise ValueError("splat takes a scalar and a count of 2, 3 or 4")
        return Value(vt_make(vt_elem(v.vt), count), v.words * count)


def U32(x: int) -> Value:
    return Value(UINT, (x & 0xFFFFFFFF,))


def I32(x: int) -> Value:
    return Value(INT, (x & 0xFFFFFFFF,))


def UVec(*xs: int) -> Value:
    return Value(vt_make("u", len(xs)), tuple(x & 0xFFFFFFFF for x in xs))


def IVec(*xs: int) -> Value:
    return Value(vt_make("i", len(xs)), tuple(x & 0xFFFFFFFF for x in xs))


def Vec2(x, y) -> Value:
    return Value.of((float(x), float(y)))


def Vec3(x, y, z) -> Value:
    return Value.of((float(x), float(y), float(z)))


def Vec4(x, y, z, w) -> Value:
    return Value.of((float(x), float(y), float(z), float(w)))


def Mat(cols: int, rows: int, data) -> Value:
    """MatrixValue::new(cols, rows, data) (reference src/graph/mod.rs:1283-1311): ``data`` holds cols*rows floats,
    column by column."""
    data = [float(x) for x in data]
    if len(data) != cols * rows:
        raise ValueError(f"a mat{cols}x{rows} takes {cols * rows} values")
    return Value(vt_matrix(cols, rows), tuple(_f32_bits(x) for x in data))


def Mat2(*cols_) -> Value:
    """From two columns (glam `Mat2::from_cols`) or four floats in column-major order."""
    return Mat(2, 2, _flatten(cols_))


def Mat3(*cols_) -> Value:
    return Mat(3, 3, _flatten(cols_))


def Mat4(*cols_) -> Value:
    return Mat(4, 4, _flatten(cols_))


def _flatten(xs):
    out = []
    for x in xs:
        out.extend(x if isinstance(x, (tuple, list)) else [x])
    return out


# ---------------------------------------------------------------------------------------------------
# Attributes (reference src/attributes.rs:1338-1378)
# ---------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class AttributeDef:
    index: int
    name: str
    vt: int
    default: Value


def _load_attributes():
    out = []
    for i in range(lib.hnb_attribute_count()):
        name, vt, words = C.c_char_p(), u32(), (u32 * 4)()
        check(lib.hnb_attribute_info(i, C.byref(name), C.byref(vt), words))
        out.append(AttributeDef(i, name.value.decode(), vt.value, Value(vt.value, tuple(words[:vt_count(vt.value)]))))
    return out


ATTRIBUTES = _load_attributes()


class Attribute:
    """Namespace of the built-in attributes: ``Attribute.POSITION`` etc."""
    ALL = ATTRIBUTES

    @staticmethod
    def by_name(name: str) -> AttributeDef:
        for a in ATTRIBUTES:
            if a.name == name:
                return a
        raise KeyError(name)


for _a in ATTRIBUTES:
    setattr(Attribute, _a.name.upper(), _a)

# operator tables (same order as the native enums / the reference's Rust enums)
BUILTINS = ["time", "delta_time", "virtual_time", "virtual_delta_time", "real_time", "real_delta_time", "rand", "alpha_cutoff", "is_alive"]
UNARY = ["abs", "acos", "asin", "atan", "all", "any", "ceil", "cos", "exp", "exp2", "floor", "fract", "inverse_sqrt", "length", "log", "log2",
         "normalize", "pack4x8snorm", "pack4x8unorm", "round", "saturate", "sign", "sin", "sqrt", "tan", "unpack4x8snorm", "unpack4x8unorm",
         "w", "x", "y", "z"]
BINARY = ["add", "atan2", "cross", "distance", "div", "dot", "gt", "ge", "lt", "le", "max", "min", "mul", "rem", "step", "sub", "uniform",
          "normal", "vec2", "vec4_xyz_w"]
TERNARY = ["mix", "clamp", "smoothstep", "vec3"]


@dataclass
class Node:
    """Recorded expression node (what the oracle interprets). ``kind`` in
    {'builtin','lit','prop','attr','parent_attr','unary','binary','ternary','cast'}."""
    kind: str
    op: str = ""
    args: tuple = ()
    value: Optional[Value] = None
    vt: int = FLOAT          # rand value type / cast target
    attr: Optional[AttributeDef] = None
    prop: str = ""


class ExprInfo(C.Structure):
    _fields_ = [("kind", u32), ("op", u32), ("value_type", u32), ("operands", u32 * 3), ("property", u32), ("attribute", C.c_char_p),
                ("literal_words", u32 * 16)]


class Module:
    """Expression module (reference src/graph/expr.rs:337). Handles are 1-based ints."""

    def __init__(self):
        self._h = lib.hnb_module_create()
        self.nodes: list[Node] = []           # nodes[h-1] mirrors native expression h
        self.properties: list[tuple[str, Value]] = []

    def __del__(self):
        try:
            if self._h:
                lib.hnb_module_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _push(self, handle: int, node: Node) -> int:
        if handle == 0:
            raise HanabiError(N.HNB_ERR_EXPR, N.last_error())
        self.nodes.append(node)
        assert handle == len(self.nodes), "native and recorded graphs out of sync"
        return handle

    def get(self, handle: int) -> ExprInfo:
        """Module::get (expr.rs:607-612): the stored expression behind a handle."""
        info = ExprInfo()
        check(lib.hnb_module_get(self._h, handle, C.byref(info)))
        return info

    def _adopt(self, handle: int) -> int:
        """Bring the recorded mirror up to date with expressions created natively (node graph lowering)."""
        if handle == 0:
            raise HanabiError(N.HNB_ERR_EXPR, N.last_error())
        for h in range(len(self.nodes) + 1, lib.hnb_module_len(self._h) + 1):
            i = self.get(h)
            a = tuple(i.operands)
            if i.kind == 0:
                node = Node("builtin", op=BUILTINS[i.op], vt=i.value_type)
            elif i.kind == 1:
                node = Node("lit", value=Value(i.value_type, tuple(i.literal_words[: vt_count(i.value_type)])))
            elif i.kind == 2:
                node = Node("prop", prop=self.properties[i.property - 1][0])
            elif i.kind in (3, 4):
                node = Node("attr" if i.kind == 3 else "parent_attr", attr=Attribute.by_name(i.attribute.decode()))
            elif i.kind == 5:
                node = Node("unary", op=UNARY[i.op], args=a[:1])
            elif i.kind == 6:
                node = Node("binary", op=BINARY[i.op], args=a[:2])
            elif i.kind == 7:
                node = Node("ternary", op=TERNARY[i.op], args=a[:3])
            else:
                node = Node("cast", args=a[:1], vt=i.value_type)
            self.nodes.append(node)
        return handle

    def lit(self, value) -> int:
        v = Value.of(value)
        words = (u32 * max(1, len(v.words)))(*v.words)
        return self._push(lib.hnb_module_lit(self._h, v.vt, words), Node("lit", value=v))

    def attr(self, a: AttributeDef) -> int:
        return self._push(lib.hnb_module_attr(self._h, a.name.encode()), Node("attr", attr=a))

    def parent_attr(self, a: AttributeDef) -> int:
        return self._push(lib.hnb_module_parent_attr(self._h, a.name.encode()), Node("parent_attr", attr=a))

    def add_property(self, name: str, default) -> int:
        v = Value.of(default)
        words = (u32 * max(1, len(v.words)))(*v.words)
        h = lib.hnb_module_add_property(self._h, name.encode(), v.vt, words)
        if h == 0:
            raise HanabiError(N.HNB_ERR_EXPR, N.last_error())
        self.properties.append((name, v))
        return h

    def prop(self, handle: int) -> int:
        name = self.properties[handle - 1][0] if 0 < handle <= len(self.properties) else "?"
        return self._push(lib.hnb_module_prop(self._h, handle), Node("prop", prop=name))

    def builtin(self, op: str, vt: int = FLOAT) -> int:
        return self._push(lib.hnb_module_builtin(self._h, BUILTINS.index(op), vt), Node("builtin", op=op, vt=vt))

    def unary(self, op: str, e: int) -> int:
        return self._push(lib.hnb_module_unary(self._h, UNARY.index(op), e), Node("unary", op=op, args=(e,)))

    def binary(self, op: str, l: int, r: int) -> int:
        return self._push(lib.hnb_module_binary(self._h, BINARY.index(op), l, r), Node("binary", op=op, args=(l, r)))

    def ternary(self, op: str, a: int, b: int, c: int) -> int:
        return self._push(lib.hnb_module_ternary(self._h, TERNARY.index(op), a, b, c), Node("ternary", op=op, args=(a, b, c)))

    def cast(self, e: int, vt: int) -> int:
        return self._push(lib.hnb_module_cast(self._h, e, vt), Node("cast", args=(e,), vt=vt))

    def get_property_by_name(self, name: str) -> Optional[int]:
        """Module::get_property_by_name: the property handle, or None."""
        for i, (n, _) in enumerate(self.properties):
            if n == name:
                return i + 1
        return None

    def is_const(self, e: int) -> bool:
        r = lib.hnb_module_is_const(self._h, e)
        if r < 0:
            raise HanabiError(r, N.last_error())
        return bool(r)

    def has_side_effect(self, e: int) -> bool:
        r = lib.hnb_module_has_side_effect(self._h, e)
        if r < 0:
            raise HanabiError(r, N.last_error())
        return bool(r)

    def eval(self, e: int, context: str = "update") -> tuple[str, str]:
        """(expression text, hoisted statements) — Expr::eval through a fresh ShaderWriter."""
        out, st = C.create_string_buffer(8192), C.create_string_buffer(8192)
        check(lib.hnb_module_eval(self._h, e, 1 if context == "init" else 2, out, 8192, st, 8192))
        return out.value.decode(), st.value.decode()


for _op in UNARY:
    setattr(Module, _op, (lambda op: lambda self, e: self.unary(op, e))(_op))
for _op in BINARY:
    setattr(Module, _op, (lambda op: lambda self, l, r: self.binary(op, l, r))(_op))
for _op in TERNARY:
    setattr(Module, _op, (lambda op: lambda self, a, b, c: self.ternary(op, a, b, c))(_op))


# ---------------------------------------------------------------------------------------------------
# Fluent API (reference ExprWriter / WriterExpr, src/graph/expr.rs:2399-4127)
# ---------------------------------------------------------------------------------------------------
def _install_module_operator_methods():
    """The reference generates one Module method per operator (`impl_module_unary!` / `_binary!` / `_ternary!`,
    expr.rs: `m.add(l, r)`, `m.normalize(e)`, `m.mix(a, b, t)` ...). Same names here, on top of unary() / binary() / ternary()."""
    for op in UNARY:
        if not hasattr(Module, op):
            setattr(Module, op, (lambda _op: lambda self, e: self.unary(_op, e))(op))
    for op in BINARY:
        if not hasattr(Module, op):
            setattr(Module, op, (lambda _op: lambda self, l, r: self.binary(_op, l, r))(op))
    for op in TERNARY:
        if not hasattr(Module, op):
            setattr(Module, op, (lambda _op: lambda self, a, b, c: self.ternary(_op, a, b, c))(op))


_install_module_operator_methods()


class WriterExpr:
    def __init__(self, writer: "ExprWriter", handle: int):
        self.writer = writer
        self.h = handle

    def expr(self) -> int:
        return self.h

    def _wrap(self, other) -> "WriterExpr":
        return other if isinstance(other, WriterExpr) else self.writer.lit(other)

    def _un(self, op):
        return WriterExpr(self.writer, self.writer.module.unary(op, self.h))

    def _bin(self, op, other):
        return WriterExpr(self.writer, self.writer.module.binary(op, self.h, self._wrap(other).h))

    def __add__(self, o): return self._bin("add", o)
    def __sub__(self, o): return self._bin("sub", o)
    def __mul__(self, o): return self._bin("mul", o)
    def __truediv__(self, o): return self._bin("div", o)
    def __mod__(self, o): return self._bin("rem", o)
    # the reference's method names for the same operators (WriterExpr::add / sub / mul / div / rem, expr.rs)
    add, sub, mul, div, rem = __add__, __sub__, __mul__, __truediv__, __mod__

    def __radd__(self, o): return self._wrap(o)._bin("add", self)
    def __rsub__(self, o): return self._wrap(o)._bin("sub", self)
    def __rmul__(self, o): return self._wrap(o)._bin("mul", self)
    def __rtruediv__(self, o): return self._wrap(o)._bin("div", self)
    def gt(self, o): return self._bin("gt", o)
    def ge(self, o): return self._bin("ge", o)
    def lt(self, o): return self._bin("lt", o)
    def le(self, o): return self._bin("le", o)
    def max(self, o): return self._bin("max", o)
    def min(self, o): return self._bin("min", o)
    def dot(self, o): return self._bin("dot", o)
    def cross(self, o): return self._bin("cross", o)
    def distance(self, o): return self._bin("distance", o)
    def atan2(self, o): return self._bin("atan2", o)
    def uniform(self, o): return self._bin("uniform", o)
    def normal(self, o): return self._bin("normal", o)
    def vec2(self, o): return self._bin("vec2", o)
    def vec4_xyz_w(self, o): return self._bin("vec4_xyz_w", o)

    def step(self, edge):
        """``x.step(edge)`` emits ``step(edge, x)`` (expr.rs:3983-3986)."""
        return self._wrap(edge)._bin("step", self)

    def mix(self, other, fraction):
        return WriterExpr(self.writer, self.writer.module.ternary("mix", self.h, self._wrap(other).h, self._wrap(fraction).h))

    def clamp(self, lo, hi):
        return WriterExpr(self.writer, self.writer.module.ternary("clamp", self.h, self._wrap(lo).h, self._wrap(hi).h))

    def smoothstep(self, lo, hi):
        """``x.smoothstep(lo, hi)`` emits ``smoothstep(lo, hi, x)`` (expr.rs:3819-3822)."""
        return WriterExpr(self.writer, self.writer.module.ternary("smoothstep", self._wrap(lo).h, self._wrap(hi).h, self.h))

    def vec3(self, y, z):
        return WriterExpr(self.writer, self.writer.module.ternary("vec3", self.h, self._wrap(y).h, self._wrap(z).h))

    def cast(self, vt: int):
        return WriterExpr(self.writer, self.writer.module.cast(self.h, vt))


for _op in UNARY:
    if not hasattr(WriterExpr, _op):
        setattr(WriterExpr, _op, (lambda op: lambda self: self._un(op))(_op))
WriterExpr.normalized = WriterExpr.normalize   # the reference's name (WriterExpr::normalized)


class ExprWriter:
    def __init__(self, module: Optional[Module] = None):
        self.module = module or Module()

    def lit(self, value) -> WriterExpr:
        return WriterExpr(self, self.module.lit(value))

    def attr(self, a: AttributeDef) -> WriterExpr:
        return WriterExpr(self, self.module.attr(a))

    def parent_attr(self, a: AttributeDef) -> WriterExpr:
        return WriterExpr(self, self.module.parent_attr(a))

    def add_property(self, name: str, default) -> int:
        return self.module.add_property(name, default)

    def prop(self, handle: int) -> WriterExpr:
        return WriterExpr(self, self.module.prop(handle))

    def push(self, expr) -> WriterExpr:
        """ExprWriter::push: wrap an expression handle of this writer's module."""
        return WriterExpr(self, _h(expr))

    def alpha_cutoff(self) -> WriterExpr:
        """BuiltInOperator::AlphaCutoff only exists in the render context; the simulation lowering rejects it at generate()."""
        return WriterExpr(self, self.module.builtin("alpha_cutoff"))

    def time(self) -> WriterExpr:
        return WriterExpr(self, self.module.builtin("time"))

    def delta_time(self) -> WriterExpr:
        return WriterExpr(self, self.module.builtin("delta_time"))

    def rand(self, vt: int = FLOAT) -> WriterExpr:
        return WriterExpr(self, self.module.builtin("rand", vt))

    def is_alive(self) -> WriterExpr:
        return WriterExpr(self, self.module.builtin("is_alive"))

    def finish(self) -> Module:
        return self.module


# ---------------------------------------------------------------------------------------------------
# Modifiers
# ---------------------------------------------------------------------------------------------------
MODIFIER_KINDS = ["", "accel", "radial_accel", "tangent_accel", "conform_to_sphere", "linear_drag", "kill_sphere", "kill_aabb",
                  "set_attribute", "inherit_attribute", "set_position_circle", "set_position_sphere", "set_position_cone3d",
                  "set_velocity_circle", "set_velocity_sphere", "set_velocity_tangent", "emit_spawn_event"]


def _h(e) -> int:
    if e is None:
        return 0
    return e.h if isinstance(e, WriterExpr) else int(e)


@dataclass
class Modifier:
    kind: str
    exprs: tuple = ()
    params: tuple = ()

    @property
    def kind_id(self) -> int:
        return MODIFIER_KINDS.index(self.kind)


def AccelModifier(accel) -> Modifier:
    return Modifier("accel", (_h(accel),))


def RadialAccelModifier(origin, accel) -> Modifier:
    return Modifier("radial_accel", (_h(origin), _h(accel)))


def TangentAccelModifier(origin, axis, accel) -> Modifier:
    return Modifier("tangent_accel", (_h(origin), _h(axis), _h(accel)))


def ConformToSphereModifier(origin, radius, influence_dist, attraction_accel, max_attraction_speed, shell_half_thickness=None,
                            sticky_factor=None) -> Modifier:
    return Modifier("conform_to_sphere", (_h(origin), _h(radius), _h(influence_dist), _h(attraction_accel), _h(max_attraction_speed),
                                          _h(shell_half_thickness), _h(sticky_factor)))


def LinearDragModifier(drag) -> Modifier:
    return Modifier("linear_drag", (_h(drag),))


def KillSphereModifier(center, sqr_radius, kill_inside: bool = False) -> Modifier:
    return Modifier("kill_sphere", (_h(center), _h(sqr_radius)), (int(kill_inside),))


def KillAabbModifier(center, half_size, kill_inside: bool = False) -> Modifier:
    return Modifier("kill_aabb", (_h(center), _h(half_size)), (int(kill_inside),))


def SetAttributeModifier(attribute: AttributeDef, value) -> Modifier:
    return Modifier("set_attribute", (_h(value),), (attribute.index,))


def InheritAttributeModifier(attribute: AttributeDef) -> Modifier:
    return Modifier("inherit_attribute", (), (attribute.index,))


SURFACE, VOLUME = 0, 1


def SetPositionCircleModifier(center, axis, radius, dimension: int = VOLUME) -> Modifier:
    return Modifier("set_position_circle", (_h(center), _h(axis), _h(radius)), (dimension,))


def SetPositionSphereModifier(center, radius, dimension: int = VOLUME) -> Modifier:
    return Modifier("set_position_sphere", (_h(center), _h(radius)), (dimension,))


def SetPositionCone3dModifier(height, base_radius, top_radius, dimension: int = VOLUME) -> Modifier:
    return Modifier("set_position_cone3d", (_h(height), _h(base_radius), _h(top_radius)), (dimension,))


def SetVelocityCircleModifier(center, axis, speed) -> Modifier:
    return Modifier("set_velocity_circle", (_h(center), _h(axis), _h(speed)))


def SetVelocitySphereModifier(center, speed) -> Modifier:
    return Modifier("set_velocity_sphere", (_h(center), _h(speed)))


def SetVelocityTangentModifier(origin, axis, speed) -> Modifier:
    return Modifier("set_velocity_tangent", (_h(origin), _h(axis), _h(speed)))


ALWAYS, ON_DIE = 0, 1


def EmitSpawnEventModifier(condition: int, count, child_index: int) -> Modifier:
    return Modifier("emit_spawn_event", (_h(count),), (condition, child_index))


# ---------------------------------------------------------------------------------------------------
# EffectAsset
# ---------------------------------------------------------------------------------------------------
GLOBAL, LOCAL = 0, 1
WHEN_VISIBLE, ALWAYS = 0, 1  # SimulationCondition (asset.rs:54-68); WhenVisible is the default
MOTION_NONE, MOTION_PRE_UPDATE, MOTION_POST_UPDATE = 0, 1, 2


@dataclass
class LayoutField:
    name: str
    vt: int
    offset: int


class EffectAsset:
    """Reference src/asset.rs:272 (simulation-relevant part): capacity, module, init/update modifiers,
    simulation space, motion integration."""

    def __init__(self, capacity: int, module: Module, name: str = "effect", simulation_space: int = GLOBAL,
                 motion_integration: int = MOTION_POST_UPDATE):
        self.name = name
        self.capacity = capacity
        self.module = module
        self.simulation_space = simulation_space
        self.motion_integration = motion_integration
        self.init_modifiers: list[Modifier] = []
        self.update_modifiers: list[Modifier] = []
        self.simulation_condition = WHEN_VISIBLE
        self._h = None

    # builder API like the reference (`.init(m)`, `.update(m)`)
    def init(self, m: Modifier) -> "EffectAsset":
        self.init_modifiers.append(m)
        self._drop_native()
        return self

    def update(self, m: Modifier) -> "EffectAsset":
        self.update_modifiers.append(m)
        self._drop_native()
        return self

    def add_modifier(self, context: str, m: Modifier) -> "EffectAsset":
        """EffectAsset::add_modifier (asset.rs:506-520): `context` is "init" or "update" (render modifiers are outside
        the simulation path); the modifier's allowed contexts are checked when the native asset is built."""
        if context not in ("init", "update"):
            raise ValueError("context must be 'init' or 'update'")
        return self.init(m) if context == "init" else self.update(m)

    def modifiers(self) -> list:
        """EffectAsset::modifiers: init modifiers, then update modifiers."""
        return list(self.init_modifiers) + list(self.update_modifiers)

    def properties(self) -> list:
        """EffectAsset::properties: (name, default value) of the module's properties."""
        return list(self.module.properties)

    def with_name(self, name: str) -> "EffectAsset":
        self.name = name
        self._drop_native()
        return self

    def with_simulation_condition(self, condition: int) -> "EffectAsset":
        """SimulationCondition (asset.rs:54): WHEN_VISIBLE / ALWAYS. Read by the host's spawner tick (spawn.rs:970-979:
        an invisible WHEN_VISIBLE effect is not ticked); it does not change the generated code."""
        self.simulation_condition = condition
        return self

    def with_simulation_space(self, space: int) -> "EffectAsset":
        self.simulation_space = space
        self._drop_native()
        return self

    def with_motion_integration(self, mode: int) -> "EffectAsset":
        self.motion_integration = mode
        self._drop_native()
        return self

    def _drop_native(self):
        if self._h:
            lib.hnb_asset_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self._drop_native()
        except Exception:
            pass

    def _native(self):
        if self._h:
            return self._h
        h = lib.hnb_asset_create(self.name.encode(), self.capacity, self.module._h)
        try:
            check(lib.hnb_asset_set_simulation_space(h, self.simulation_space))
            check(lib.hnb_asset_set_motion_integration(h, self.motion_integration))
            for ctx, mods in ((1, self.init_modifiers), (2, self.update_modifiers)):
                for m in mods:
                    ex = (u32 * max(1, len(m.exprs)))(*m.exprs)
                    pa = (u32 * max(1, len(m.params)))(*m.params)
                    check(lib.hnb_asset_add_modifier(h, ctx, m.kind_id, ex, len(m.exprs), pa, len(m.params)))
        except Exception:
            lib.hnb_asset_destroy(h)
            raise
        self._h = h
        return h

    def particle_layout(self) -> tuple[list[LayoutField], int, int]:
        """(fields incl. pads in offset order, size bytes, align) — EffectAsset::particle_layout."""
        arr = (N.AttrLayout * 64)()
        n, size, align = u32(), u32(), u32()
        check(lib.hnb_asset_particle_layout(self._native(), arr, 64, C.byref(n), C.byref(size), C.byref(align)))
        return [LayoutField(arr[i].name.decode(), arr[i].value_type, arr[i].offset) for i in range(n.value)], size.value, align.value

    def property_layout(self) -> tuple[list[LayoutField], int]:
        arr = (N.AttrLayout * 64)()
        n, size = u32(), u32()
        check(lib.hnb_asset_property_layout(self._native(), arr, 64, C.byref(n), C.byref(size)))
        return [LayoutField(arr[i].name.decode(), arr[i].value_type, arr[i].offset) for i in range(n.value)], size.value

    def serialize_properties(self, values: dict | None = None) -> bytes:
        values = values or {}
        names = (C.c_char_p * max(1, len(values)))(*[k.encode() for k in values])
        bufs = []
        for v in values.values():
            val = Value.of(v)
            bufs.append((u32 * max(1, len(val.words)))(*val.words))
        ptrs = (P(u32) * max(1, len(values)))(*[C.cast(b, P(u32)) for b in bufs])
        size = u32()
        check(lib.hnb_asset_serialize_properties(self._native(), names, ptrs, len(values), None, 0, C.byref(size)))
        blob = C.create_string_buffer(max(1, size.value))
        check(lib.hnb_asset_serialize_properties(self._native(), names, ptrs, len(values), blob, size.value, C.byref(size)))
        return blob.raw[:size.value]

    def generate(self, parent: Optional["EffectAsset"] = None, num_event_bindings: int = 0, relaxed_order: bool = False,
                 fast_math: bool = False, ordered_events: bool = False, sector_planes: bool = False, slot_order: bool = False) -> LoweredEffect:
        """EffectShaderSources::generate: lower to the Level-1 effect description."""
        g = C.c_void_p()
        check(lib.hnb_asset_generate(self._native(), parent._native() if parent else None, num_event_bindings, C.byref(g)))
        try:
            d = N.EffectDesc()
            check(lib.hnb_generated_desc(g, C.byref(d)))

            def s(x):
                return x.decode() if x else ""

            fx = LoweredEffect(
                name=s(d.name), attrs=[AttrField(s(d.attrs[i].name), d.attrs[i].value_type, d.attrs[i].offset, d.attrs[i].flags)
                                            for i in range(d.n_attrs)],
                particle_stride=d.particle_stride, init_code=s(d.init_code), init_extra=s(d.init_extra), sim_space_code=s(d.sim_space_code),
                age_code=s(d.age_code), reap_code=s(d.reap_code), update_code=s(d.update_code), update_extra=s(d.update_extra),
                properties_struct=s(d.properties_struct), properties_size=d.properties_size,
                flags=d.flags | (N.EFFECT_RELAXED_ORDER if relaxed_order else 0) | (N.EFFECT_FAST_MATH if fast_math else 0)
                | (N.EFFECT_ORDERED_EVENTS if ordered_events else 0) | (N.EFFECT_SECTOR_PLANES if sector_planes else 0)
                | (N.EFFECT_SLOT_ORDER if slot_order else 0),
                parent_attrs=[AttrField(s(d.parent_attrs[i].name), d.parent_attrs[i].value_type, d.parent_attrs[i].offset) for i in range(d.n_parent_attrs)],
                parent_particle_stride=d.parent_particle_stride, num_event_bindings=d.num_event_bindings)
        finally:
            lib.hnb_generated_destroy(g)
        return fx


# ---------------------------------------------------------------------------------------------------
# Node-graph front end (reference src/graph/node.rs)
# ---------------------------------------------------------------------------------------------------
NODE_ADD, NODE_SUB, NODE_MUL, NODE_DIV, NODE_ATTRIBUTE, NODE_TIME, NODE_NORMALIZE = range(1, 8)


@dataclass(frozen=True)
class NodeSpec:
    kind: int
    attribute: Optional[str] = None


def AddNode() -> NodeSpec: return NodeSpec(NODE_ADD)
def SubNode() -> NodeSpec: return NodeSpec(NODE_SUB)
def MulNode() -> NodeSpec: return NodeSpec(NODE_MUL)
def DivNode() -> NodeSpec: return NodeSpec(NODE_DIV)
def TimeNode() -> NodeSpec: return NodeSpec(NODE_TIME)
def NormalizeNode() -> NodeSpec: return NodeSpec(NODE_NORMALIZE)


def AttributeNode(attr: Optional[AttributeDef] = None) -> NodeSpec:
    return NodeSpec(NODE_ATTRIBUTE, attr.name if attr is not None else None)


@dataclass
class SlotInfo:
    name: str
    node: int
    is_input: bool
    value_type: Optional[int]
    linked: list


class Graph:
    """Graph (node.rs:244-443): nodes, slots and links; NodeId / SlotId are the reference's 1-based ids."""

    def __init__(self):
        self._h = lib.hnb_node_graph_create()

    def __del__(self):
        try:
            if self._h:
                lib.hnb_node_graph_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def add_node(self, node: NodeSpec) -> int:
        nid = lib.hnb_node_graph_add_node(self._h, node.kind, node.attribute.encode() if node.attribute else None)
        if not nid:
            raise N.HanabiError(N.HNB_ERR_EXPR, N.last_error())
        return nid

    def link(self, output: int, input: int):
        check(lib.hnb_node_graph_link(self._h, output, input))

    def unlink(self, output: int, input: int):
        check(lib.hnb_node_graph_unlink(self._h, output, input))

    def unlink_all(self, slot: int):
        check(lib.hnb_node_graph_unlink_all(self._h, slot))

    def _slots(self, node: int, direction: int) -> list:
        arr, n = (u32 * 8)(), u32()
        check(lib.hnb_node_graph_slots(self._h, node, direction, arr, 8, C.byref(n)))
        return list(arr[: n.value])

    def slots(self, node: int) -> list: return self._slots(node, 0)
    def input_slots(self, node: int) -> list: return self._slots(node, 1)
    def output_slots(self, node: int) -> list: return self._slots(node, 2)

    def input_slot(self, node: int, name: str) -> Optional[int]:
        return lib.hnb_node_graph_find_slot(self._h, node, 1, name.encode()) or None

    def output_slot(self, node: int, name: str) -> Optional[int]:
        return lib.hnb_node_graph_find_slot(self._h, node, 2, name.encode()) or None

    def get_slot_id(self, name: str) -> Optional[int]:
        return lib.hnb_node_graph_find_slot(self._h, 0, 0, name.encode()) or None

    def slot(self, slot: int) -> SlotInfo:
        name, node, is_in, vt, linked, n = C.c_char_p(), u32(), u32(), C.c_int32(), (u32 * 64)(), u32()
        check(lib.hnb_node_graph_slot_info(self._h, slot, C.byref(name), C.byref(node), C.byref(is_in), C.byref(vt), linked, 64, C.byref(n)))
        return SlotInfo(name.value.decode(), node.value, bool(is_in.value), None if vt.value < 0 else vt.value, list(linked[: n.value]))

    def eval_node(self, node: int, module: "Module", inputs: Sequence[int]) -> list:
        """Node::eval: handles of the node's outputs in `module`."""
        arr = (u32 * max(1, len(inputs)))(*inputs)
        out, n = (u32 * 4)(), u32()
        check(lib.hnb_node_graph_eval_node(self._h, node, module._h, arr, len(inputs), out, 4, C.byref(n)))
        return [module._adopt(h) for h in out[: n.value]]

    def eval_slot(self, module: "Module", output_slot: int) -> int:
        """Lower everything `output_slot` depends on; returns the expression handle."""
        out = u32()
        check(lib.hnb_node_graph_eval_slot(self._h, module._h, output_slot, C.byref(out)))
        return module._adopt(out.value)


@dataclass
class PropertyInstance:
    """PropertyInstance (properties.rs:183-190): definition (name, default) and current value."""
    name: str
    default_value: Value
    value: Value


class EffectProperties:
    """Per-instance property values (reference src/properties.rs:205-454): what `hnb_upload_properties` receives is
    `serialize(asset)`. Method names follow the reference; where it asserts, HanabiError is raised."""

    def __init__(self):
        self._h = lib.hnb_effect_properties_create()

    def __del__(self):
        try:
            if self._h:
                lib.hnb_effect_properties_destroy(self._h)
                self._h = None
        except Exception:
            pass

    @staticmethod
    def _words(v: Value):
        return (u32 * 16)(*v.words)

    def with_properties(self, properties) -> "EffectProperties":
        for name, value in properties:
            self.set(name, value)
        return self

    def set(self, name: str, value) -> None:
        v = Value.of(value)
        check(lib.hnb_effect_properties_set(self._h, name.encode(), v.vt, self._words(v)))

    def set_if_changed(self, name: str, value) -> bool:
        v = Value.of(value)
        changed = u32()
        check(lib.hnb_effect_properties_set_if_changed(self._h, name.encode(), v.vt, self._words(v), C.byref(changed)))
        return bool(changed.value)

    def get_stored(self, name: str) -> Optional[Value]:
        vt, words = u32(), (u32 * 16)()
        if not lib.hnb_effect_properties_get_stored(self._h, name.encode(), C.byref(vt), words):
            return None
        return Value(vt.value, tuple(words[: vt_count(vt.value)]))

    def properties(self) -> list:
        out = []
        for i in range(lib.hnb_effect_properties_len(self._h)):
            name, vt, val, dflt = C.c_char_p(), u32(), (u32 * 16)(), (u32 * 16)()
            check(lib.hnb_effect_properties_get(self._h, i, C.byref(name), C.byref(vt), val, dflt))
            n = vt_count(vt.value)
            out.append(PropertyInstance(name.value.decode(), Value(vt.value, tuple(dflt[:n])), Value(vt.value, tuple(val[:n]))))
        return out

    def update(self, asset: "EffectAsset") -> bool:
        """EffectProperties::update against the asset's properties; returns whether the store changed."""
        changed = u32()
        check(lib.hnb_effect_properties_update(self._h, asset._native(), C.byref(changed)))
        return bool(changed.value)

    def serialize(self, asset: "EffectAsset") -> bytes:
        size = u32()
        check(lib.hnb_effect_properties_serialize(self._h, asset._native(), None, 0, C.byref(size)))
        blob = C.create_string_buffer(max(1, size.value))
        check(lib.hnb_effect_properties_serialize(self._h, asset._native(), blob, size.value, C.byref(size)))
        return blob.raw[:size.value]


def particle_layout_of(names: Sequence[str]) -> tuple[list[LayoutField], int, int]:
    """ParticleLayout::new().append(..).build() for a list of attribute names."""
    arr_names = (C.c_char_p * max(1, len(names)))(*[n.encode() for n in names])
    arr = (N.AttrLayout * 64)()
    n, size, align = u32(), u32(), u32()
    check(lib.hnb_particle_layout_build(arr_names, len(names), arr, 64, C.byref(n), C.byref(size), C.byref(align)))
    return [LayoutField(arr[i].name.decode(), arr[i].value_type, arr[i].offset) for i in range(n.value)], size.value, align.value


def format_f32(x: float) -> str:
    buf = C.create_string_buffer(64)
    check(lib.hnb_format_f32(x, buf, 64))
    return buf.value.decode()
