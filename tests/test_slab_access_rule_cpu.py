"""What each host call enqueues before it touches a slab, on the CPU: bevy_hanabi_b200/csrc/runtime/slab_access_rule.h
compiled with g++ and called through ctypes, held to the writer / reader tables of DESIGN.md §3, restated here.

A slab keeps two identity claims, a lifetime floor and a common-age word per 32 rows, and host flags: whether an update may
have left words deferred (`defers`), whether updates get floors or ages at all, and whether records were written before the
column plan was fixed. For each entry point the tables say whether the claims are dropped, and what happens to the group
words of the rows: nothing, a flush that writes deferred ages back (readers), or a flush and the sentinel (writers), over the
call's rows or the whole slab. On a slab that never deferred a writer sets the sentinel with memsets and a reader does
nothing.
"""
import ctypes as C
import hashlib
import random
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "build" / "slab_access_rule"
RULE_H = ROOT / "bevy_hanabi_b200" / "csrc" / "runtime" / "slab_access_rule.h"

KINDS = ["RecordRead", "RecordWrite", "RowReset", "ListWrite", "AliveBitsWrite", "InstanceRewrite", "Append", "Invalidate",
         "MetadataWrite", "ViewOut", "Bind", "DeferringUpdate", "ListSort"]

RULE_DRIVER = r"""
#include <cstring>
#include "slab_access_rule.h"
using namespace hnb_rt;
extern "C" int rule_kind(const char* name) {
#define K(x) if (!strcmp(name, #x)) return int(SlabAccess::x);
    K(RecordRead) K(RecordWrite) K(RowReset) K(ListWrite) K(AliveBitsWrite) K(InstanceRewrite) K(Append) K(Invalidate)
    K(MetadataWrite) K(ViewOut) K(Bind) K(DeferringUpdate) K(ListSort)
#undef K
    return -1;
}
extern "C" void rule_sizes(uint32_t* out) { out[0] = sizeof(SlabState); out[1] = sizeof(ModuleWords); out[2] = sizeof(SlabWork); }
extern "C" void rule_access(SlabState* s, int kind, uint32_t first, uint32_t count, uint32_t capacity, const ModuleWords* m,
                            SlabWork* out) {
    *out = slab_access(*s, SlabAccess(kind), first, count, capacity, *m);
}
extern "C" int rule_keeps_group_ages(const SlabState* s) { return keeps_group_ages(*s) ? 1 : 0; }
"""


class State(C.Structure):
    _fields_ = [("plan_fixed", C.c_bool), ("written", C.c_bool), ("floors_off", C.c_bool), ("ages_off", C.c_bool),
                ("defers", C.c_bool), ("age_word", C.c_uint32)]

    def flags(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


class Module(C.Structure):
    _fields_ = [("life_floor", C.c_bool), ("group_age", C.c_bool), ("age_word", C.c_uint32)]


class Work(C.Structure):
    _fields_ = [("drop_claims", C.c_bool), ("flush", C.c_bool), ("clear", C.c_bool), ("first", C.c_uint32), ("count", C.c_uint32)]

    def tuple(self):
        return (self.drop_claims, self.flush, self.clear, self.first, self.count)


@pytest.fixture(scope="module")
def rule():
    text = RULE_DRIVER + "// " + hashlib.sha1(RULE_H.read_bytes()).hexdigest() + "\n"
    OUT.mkdir(parents=True, exist_ok=True)
    tag = hashlib.sha1(text.encode()).hexdigest()[:16]
    cpp, so = OUT / f"rule_{tag}.cpp", OUT / f"rule_{tag}.so"
    if not so.exists():
        cpp.write_text(text)
        tmp = f"{so}.{id(text)}.tmp"
        proc = subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-Wall", "-Werror", "-I", str(RULE_H.parent), str(cpp), "-o", tmp],
                              capture_output=True, text=True)
        assert proc.returncode == 0, proc.stderr[:4000]
        Path(tmp).replace(so)
    lib = C.CDLL(str(so))
    lib.rule_kind.argtypes, lib.rule_kind.restype = [C.c_char_p], C.c_int
    lib.rule_access.argtypes = [C.POINTER(State), C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(Module), C.POINTER(Work)]
    lib.rule_access.restype = None
    lib.rule_keeps_group_ages.argtypes, lib.rule_keeps_group_ages.restype = [C.POINTER(State)], C.c_int
    sizes = (C.c_uint32 * 3)()
    lib.rule_sizes(sizes)
    assert list(sizes) == [C.sizeof(State), C.sizeof(Module), C.sizeof(Work)], "ctypes mirrors of the rule's structs"
    lib.kind = {k: lib.rule_kind(k.encode()) for k in KINDS}
    assert -1 not in lib.kind.values() and len(set(lib.kind.values())) == len(KINDS)
    return lib


def access(rule, state, kind, first=0, count=0, cap=9173, module=None):
    w = Work()
    rule.rule_access(C.byref(state), rule.kind[kind], first, count, cap, C.byref(module or Module()), C.byref(w))
    return w


CAP = 9173
ROWS = (70, 1000)  # starts and ends inside a 32-row group

# ---- DESIGN.md §3, restated: entry point -> (access kind, drops the claims, group words, scope) ------------------------
#  group words: None (untouched), "read" (deferred ages written back, the words stay known), "clear" (written back, then
#  the sentinel), "materialise" (written back and the sentinel, on a slab that may defer; nothing otherwise)
#  scope: "rows" (the groups of the call's rows), "whole" (the whole slab), "list" (the whole slab when it may defer, the
#  groups of the positions otherwise)
ENTRY_POINTS = {
    "hnb_slab_create": ("RowReset", True, "clear", "rows"),  # all rows of the new slab
    "hnb_slab_reset_rows": ("RowReset", True, "clear", "rows"),
    "hnb_slab_fill_c5": ("RecordWrite", False, "clear", "rows"),
    "hnb_slab_upload_aos": ("RecordWrite", False, "clear", "rows"),
    "hnb_slab_import_aos_device": ("RecordWrite", False, "clear", "rows"),
    "hnb_slab_upload_indirect": ("ListWrite", True, "clear", "list"),
    "hnb_slab_import_indirect_device": ("ListWrite", True, "clear", "list"),
    "hnb_slab_rebuild_alive_bits": ("AliveBitsWrite", False, "clear", "list"),
    "hnb_slab_repack": ("InstanceRewrite", False, "clear", "rows"),
    "hnb_instance_restore": ("InstanceRewrite", False, "clear", "rows"),
    "hnb_instance_append": ("Append", False, None, "rows"),
    "30-bit epoch wrap": ("Invalidate", False, "clear", "whole"),
    "plan migration": ("Invalidate", False, "clear", "whole"),
    "hnb_metadata_insert": ("MetadataWrite", False, "materialise", "whole"),
    "hnb_slab_download_aos": ("RecordRead", False, "read", "rows"),
    "hnb_slab_export_aos_device": ("RecordRead", False, "read", "rows"),
    "hnb_instance_snapshot": ("RecordRead", False, "read", "rows"),
    "hnb_slab_checksum": ("RecordRead", False, "read", "rows"),
    "ribbon sort": ("ListSort", True, "read", "whole"),
    "hnb_slab_device_view": ("ViewOut", False, "materialise", "whole"),
}
WRITES_RECORDS_BEFORE_PLAN = {"RecordWrite"}  # what marks a slab `written` (repack, restore, append fix the plan first)


def expected(groups, scope, claims, defers, first, count, cap):
    """(drop_claims, flush, clear, first, count) the tables ask for."""
    whole = scope == "whole" or (scope == "list" and defers and count)
    f, n = (0, cap) if whole else (first, count)
    if groups is None or n == 0 or (groups == "materialise" and not defers):
        return (claims, False, False, 0, 0)
    if groups == "read":
        return (claims, True, False, f, n) if defers else (claims, False, False, 0, 0)
    return (claims, defers, True, f, n)


@pytest.mark.parametrize("defers", [False, True], ids=["never-deferred", "defers"])
@pytest.mark.parametrize("entry", sorted(ENTRY_POINTS))
@pytest.mark.parametrize("rows", [ROWS, (0, CAP), (CAP - 1, 1), (500, 0)], ids=["range", "all-rows", "last-row", "no-rows"])
def test_entry_point_against_the_tables(rule, entry, defers, rows):
    kind, claims, groups, scope = ENTRY_POINTS[entry]
    if entry == "hnb_slab_create":
        rows = (0, CAP)
    s = State(defers=defers, age_word=3, plan_fixed=False)
    before = s.flags()
    w = access(rule, s, kind, *rows, cap=CAP)
    want = expected(groups, scope, claims, defers, *rows, CAP)
    assert w.tuple() == want, f"{entry} ({kind}) on a slab that {'defers' if defers else 'never deferred'}, rows {rows}"
    after = dict(before)
    if kind in WRITES_RECORDS_BEFORE_PLAN:
        after["written"] = True
    if kind == "ViewOut":
        after["floors_off"] = True           # records written through the view would not clear the floors
    if want[1] and want[2] and (want[3], want[4]) == (0, CAP):
        after["defers"] = False              # a whole-slab clear leaves no word deferred
    assert s.flags() == after, entry


# ---- binds: a module with floors and ages in the slab's age word keeps them; any other clears the slab for good ---------
MODULES = {
    "floors and ages, same word": (Module(life_floor=True, group_age=True, age_word=3), False, False, False),
    "floors and ages, other word": (Module(life_floor=True, group_age=True, age_word=5), True, False, False),
    "floors only": (Module(life_floor=True, group_age=False), True, False, True),
    "no floors (relaxed / slot order)": (Module(), True, True, True),
}


@pytest.mark.parametrize("defers", [False, True], ids=["never-deferred", "defers"])
@pytest.mark.parametrize("name", sorted(MODULES))
def test_bind(rule, name, defers):
    m, materialises, floors_off, ages_off = MODULES[name]
    s = State(defers=defers, age_word=3)
    w = access(rule, s, "Bind", 0, 0, cap=CAP, module=m)
    assert w.tuple() == ((False, True, True, 0, CAP) if defers and materialises else (False, False, False, 0, 0))
    assert (s.floors_off, s.ages_off) == (floors_off, ages_off)
    assert s.defers == (defers and not materialises)
    assert bool(rule.rule_keeps_group_ages(C.byref(s))) == (not floors_off and not ages_off)
    # the flags are permanent: a later bind of a module that keeps both words does not bring them back
    access(rule, s, "Bind", module=Module(life_floor=True, group_age=True, age_word=3))
    assert (s.floors_off, s.ages_off) == (floors_off, ages_off)


def test_deferring_update(rule):
    s = State(age_word=3)
    w = access(rule, s, "DeferringUpdate", module=Module(life_floor=True, group_age=True, age_word=7))
    assert w.tuple() == (False, False, False, 0, 0)
    assert s.defers and s.age_word == 7
    # a reader then flushes with that word's slab state, and a partial clear keeps the slab deferring
    assert access(rule, s, "RecordWrite", *ROWS).tuple() == (False, True, True, *ROWS) and s.defers
    assert access(rule, s, "RecordWrite", 0, CAP).tuple() == (False, True, True, 0, CAP) and not s.defers


# ---- flag transitions over random call sequences ---------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_flag_transitions(rule, seed):
    """`defers` goes up only in a deferring update and down only with a whole-slab clear; `floors_off` and `ages_off` never
    go down; `written` goes up only with a record writer; every returned work matches the tables."""
    rng = random.Random(seed)
    by_kind = {}
    for entry, spec in ENTRY_POINTS.items():
        by_kind.setdefault(spec[0], spec)
    s = State(age_word=3)
    seen = set()
    for _ in range(4000):
        kind = rng.choice(KINDS)
        first = rng.randrange(CAP)
        count = rng.choice([0, 1, rng.randrange(CAP - first + 1), CAP - first])
        if rng.random() < 0.1:
            first, count = 0, CAP
        m = Module(life_floor=rng.random() < 0.9, group_age=rng.random() < 0.9, age_word=rng.choice([3, 3, 3, 5]))
        if kind == "DeferringUpdate" and not rule.rule_keeps_group_ages(C.byref(s)):
            continue  # launch_update asks only when updates keep the ages
        before = s.flags()
        w = access(rule, s, kind, first, count, cap=CAP, module=m)
        after = s.flags()
        if kind in by_kind:
            _, claims, groups, scope = by_kind[kind]
            assert w.tuple() == expected(groups, scope, claims, before["defers"], first, count, CAP), (kind, first, count, before)
        whole_clear = w.flush and w.clear and (w.first, w.count) == (0, CAP)
        if after["defers"] and not before["defers"]:
            assert kind == "DeferringUpdate"
        if before["defers"] and not after["defers"]:
            assert whole_clear, kind
        if before["defers"] and whole_clear:
            assert not after["defers"]
        for f in ("floors_off", "ages_off", "written"):
            assert after[f] >= before[f], (kind, f)
        if after["written"] != before["written"]:
            assert kind in WRITES_RECORDS_BEFORE_PLAN
        assert after["plan_fixed"] == before["plan_fixed"]  # only fix_plan fixes the plan
        seen.add((kind, before["defers"], w.flush, w.clear))
        if rng.random() < 0.02:
            s = State(age_word=3)
    assert {k for k, *_ in seen} == set(KINDS)
    assert any(d and fl and cl for _, d, fl, cl in seen) and any(not d and not fl and cl for _, d, fl, cl in seen)
