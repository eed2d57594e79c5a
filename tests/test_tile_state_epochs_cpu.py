"""The update look-back's tile states from one frame to the next, on the CPU and deterministic.

A batch slot keeps its array of tile state words from frame to frame: hnb_update reads a predecessor's word and takes it as
published this frame when its epoch tag equals the frame's (`hnb_state_flag`). Slot-order words keep 6 bits of epoch,
default-order words 30 (relaxed order runs no look-back). So a word written 64 frames earlier, or any multiple, passes
for current in slot order whenever the tile that wrote it was not rewritten since: the batch slot sat out, or served
another instance with fewer tiles. The host zeroes an array before such a run (bevy_hanabi_b200/csrc/runtime/
tile_state_rule.h, called by bind_launch).

This model keeps one persistent state array per batch slot across frames, with per-frame geometry, and runs:
  * the real state words: `hnb_pack_state` / `hnb_state_flag` of the kernel header, from the g++ build tests/kernel_emu.py
    makes of a slot-order and of a default-order effect;
  * the real host rule: tile_state_rule.h compiled with g++, called through ctypes, in the order context.cpp calls it
    (plan every batch of the frame, then next_epoch with its 30-bit wrap, then the update runs);
  * an adversarial schedule: a tile looks back BEFORE its predecessors publish whenever the protocol lets it, so an old
    word that passes for current is consumed. Every word also records, outside the 64 bits, the frame that wrote it:
    consuming an older one fails with "stale".
The GPU suite (tests/test_gpu_batch_slots.py) runs the same situations on the device, where they depend on timing.
"""
import ctypes as C
import hashlib
import random
import subprocess
from pathlib import Path

import pytest

from bevy_hanabi_b200 import recipes
from tests.kernel_emu import build_emulated_effect

ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "build" / "tile_state_rule"
RULE_H = ROOT / "bevy_hanabi_b200" / "csrc" / "runtime" / "tile_state_rule.h"
WINDOW = 32            # predecessors per look-back window (hnb_compact_tile)
AGGREGATE, PREFIX = 1, 2
EPOCH_MASK = 0x3FFFFFFF

pytestmark = pytest.mark.timeout(900)

RULE_DRIVER = r"""
#include "tile_state_rule.h"
extern "C" uint32_t rule_run_epoch(uint32_t epoch) { return hnb_rt::tile_state_run_epoch(epoch); }
extern "C" int rule_needs_clear(uint64_t* sig, uint32_t* first_epoch, uint64_t new_sig, uint32_t run_epoch) {
    hnb_rt::TileStateSlot s;
    s.sig = *sig;
    s.first_epoch = *first_epoch;
    const bool clear = hnb_rt::tile_state_needs_clear(s, new_sig, run_epoch);
    *sig = s.sig;
    *first_epoch = s.first_epoch;
    return clear ? 1 : 0;
}
"""


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
    lib.rule_run_epoch.argtypes, lib.rule_run_epoch.restype = [C.c_uint32], C.c_uint32
    lib.rule_needs_clear.argtypes = [C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.c_uint64, C.c_uint32]
    lib.rule_needs_clear.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def words():
    """The kernel's state word functions per order: {"slot": lib, "default": lib}."""
    return {"slot": build_emulated_effect(recipes.c5_lowered(slot_order=True)), "default": build_emulated_effect(recipes.c5_lowered())}


class RealRule:
    """bind_launch's decision through the compiled header."""

    def __init__(self, lib):
        self.lib = lib
        self.slots = {}

    def run_epoch(self, epoch):
        return self.lib.rule_run_epoch(epoch)

    def reset(self, slot):
        self.slots[slot] = (C.c_uint64(0), C.c_uint32(0))

    def needs_clear(self, slot, sig, run_epoch):
        s, f = self.slots.setdefault(slot, (C.c_uint64(0), C.c_uint32(0)))
        return bool(self.lib.rule_needs_clear(C.byref(s), C.byref(f), sig, run_epoch))


class SignatureOnlyRule(RealRule):
    """The rule before the 64-frame limit, restated: zero a batch's array only when its signature changes."""

    def needs_clear(self, slot, sig, run_epoch):
        old = self.slots.get(slot, 0)
        self.slots[slot] = sig
        return sig != old

    def reset(self, slot):
        self.slots[slot] = 0


class Context:
    """The host side of hnb_simulate for the tile states: per batch slot one persistent array, the epoch, the rule."""

    def __init__(self, words, rule, epoch_start=0, rng=None, cap=64):
        self.words, self.rule, self.epoch, self.cap = words, rule, epoch_start & EPOCH_MASK, cap
        self.arrays = {}           # slot -> [word]
        self.writer = {}           # slot -> [epoch of the run that wrote the word, or None]
        self.rng = rng or random.Random(0)
        self.clears = 0
        self.frame_no = 0

    def _array(self, slot):
        if slot not in self.arrays:                           # ensure_tile_state: a new array is zeroed and its record reset
            self.arrays[slot], self.writer[slot] = [0] * self.cap, [None] * self.cap
            self.rule.reset(slot)
        return self.arrays[slot], self.writer[slot]

    def _zero(self, slot):
        self.arrays[slot][:] = [0] * self.cap
        self.writer[slot][:] = [None] * self.cap

    def frame(self, batches, schedule="adversarial"):
        """batches: [(slot, use)], use = dict(order="slot"|"default", sig=<what bind_launch hashes>, alive=[[per-tile survivors]
        per instance], valid=[[per-tile valid rows]]). Returns {slot: [exclusive prefix per tile]}."""
        self.frame_no += 1
        run = self.rule.run_epoch(self.epoch)
        for slot, use in batches:                             # bind_launch, before next_epoch
            self._array(slot)
            sig = use["sig"] if use["order"] == "slot" else 0
            if self.rule.needs_clear(slot, sig, run):
                self._zero(slot)
                self.clears += 1
        self.epoch = (self.epoch + 1) & EPOCH_MASK            # next_epoch
        if self.epoch == 0:
            self.epoch = 1
            for slot in self.arrays:
                self._zero(slot)
        assert self.epoch == run
        return {slot: self._run(slot, use, schedule) for slot, use in batches}

    def _run(self, slot, use, schedule):
        lib = self.words[use["order"]]
        states, writer = self._array(slot)
        alive, inst_first = [], []
        for tiles in use["alive"]:
            first = len(alive)
            alive += tiles
            inst_first += [first] * len(tiles)
        valid = [v for tiles in use.get("valid", use["alive"]) for v in tiles]
        total = len(alive)
        assert total <= self.cap
        epoch = self.epoch
        published = [False] * total
        exclusive = [None] * total

        def publish(t, flag, survivors, vld):
            states[t] = lib.emu_pack_state(epoch, flag, survivors, vld)
            writer[t] = epoch

        def counts(word):
            v = lib.emu_state_value(word)
            if use["order"] == "slot":
                return v >> 28, v & 0xFFFFFFF
            return v, 0

        def resolve(t):
            """hnb_compact_tile's look-back for tile t; a needed predecessor that has not published makes the tile wait,
            which the adversary resolves by running that predecessor first."""
            first = inst_first[t]
            if t == first:
                exclusive[t] = (0, 0)
                return
            sur, vld, pos = 0, 0, t - 1
            while True:
                window = []
                for back in range(WINDOW):
                    p = pos - back
                    window.append((p, states[p]) if p >= first else (p, lib.emu_pack_state(epoch, PREFIX, 0, 0)))
                need = []
                for p, w in window:
                    need.append((p, w))
                    if lib.emu_state_flag(w, epoch) == PREFIX:
                        break
                waiting = [p for p, w in need if lib.emu_state_flag(w, epoch) == 0]
                if waiting:
                    step(waiting[0])                          # poll: the nearest unpublished predecessor runs
                    continue
                for p, w in need:
                    if p >= first and writer[p] != epoch:
                        raise AssertionError(f"stale tile state consumed: frame epoch {epoch}, tile {t} read tile {p}'s word of epoch {writer[p]}")
                    s, v = counts(w)
                    sur, vld = sur + s, vld + v
                if lib.emu_state_flag(need[-1][1], epoch) == PREFIX:
                    break
                pos -= WINDOW
            exclusive[t] = (sur, vld)
            publish(t, PREFIX, sur + alive[t], vld + valid[t])

        def step(t):
            """Tile t's pass 1 (publish AGGREGATE, or PREFIX for an instance's first tile), then its look-back."""
            if published[t]:
                return
            published[t] = True
            publish(t, PREFIX if t == inst_first[t] else AGGREGATE, alive[t], valid[t])
            resolve(t)

        order = list(range(total - 1, -1, -1))                 # every tile looks back before its predecessors publish
        if schedule == "random":
            self.rng.shuffle(order)
        for t in order:
            step(t)
        run_s, run_v, want = 0, 0, []
        for t in range(total):
            if inst_first[t] == t:
                run_s = run_v = 0
            want.append((run_s, run_v if use["order"] == "slot" else 0))
            run_s, run_v = run_s + alive[t], run_v + valid[t]
        assert exclusive == want, f"epoch {epoch}: exclusive prefixes {exclusive} != {want}"
        return exclusive


def _use(order, sig, tiles, rng, max_count=128):
    alive = [[rng.randint(0, max_count) for _ in range(n)] for n in tiles]
    return dict(order=order, sig=sig, alive=alive, valid=[[rng.randint(a, max_count) for a in inst] for inst in alive])


# ---- the state words themselves ----------------------------------------------------------------------------------------
def test_state_word_epoch_width(words):
    """Slot-order words match any epoch congruent mod 64; default-order words the exact 30-bit epoch. A zero word is
    never published."""
    s, d = words["slot"], words["default"]
    for e in (1, 2, 63, 64, 65, 1000, EPOCH_MASK - 1, EPOCH_MASK):
        ws = s.emu_pack_state(e, PREFIX, 5, 7)
        assert s.emu_state_flag(ws, e) == PREFIX
        assert s.emu_state_flag(ws, e + 64) == PREFIX and s.emu_state_flag(ws, e + 128) == PREFIX
        assert s.emu_state_flag(ws, e + 1) == 0 and s.emu_state_flag(ws, e + 63) == 0
        wd = d.emu_pack_state(e, AGGREGATE, 5, 0)
        assert d.emu_state_flag(wd, e) == AGGREGATE
        assert d.emu_state_flag(wd, (e + 64) & EPOCH_MASK) == 0 and d.emu_state_flag(wd, (e + (1 << 24)) & EPOCH_MASK) == 0
        for lib in (s, d):
            assert lib.emu_state_flag(0, e) == 0
    assert s.emu_state_value(s.emu_pack_state(9, PREFIX, (1 << 28) - 1, (1 << 28) - 2)) == (((1 << 28) - 1) << 28) | ((1 << 28) - 2)


def test_run_epoch_follows_next_epoch(rule):
    assert rule.rule_run_epoch(0) == 1 and rule.rule_run_epoch(41) == 42
    assert rule.rule_run_epoch(EPOCH_MASK - 1) == EPOCH_MASK
    assert rule.rule_run_epoch(EPOCH_MASK) == 1          # 0 is skipped at the wrap


# ---- the two scenarios, old rule against the real one ------------------------------------------------------------------
def _sit_out(ctx, gap, rng):
    """X in slot 0 every frame; Y (same effect and slab, so the same signature on return) in slot 1, absent for `gap`."""
    x, y = _use("slot", 11, [3], rng), _use("slot", 22, [4], rng)
    ctx.frame([(0, x), (1, y)])
    for _ in range(gap):
        ctx.frame([(0, _use("slot", 11, [3], rng))])
    ctx.frame([(0, x), (1, _use("slot", 22, [4], rng))])


def _hand_over(ctx, frames_y, rng):
    """Slot 0 serves X (4 tiles) at one frame, then Y (2 tiles, same effect / slab / tile word: the same signature) for
    `frames_y` frames, then X again."""
    ctx.frame([(0, _use("slot", 7, [4], rng))])
    for _ in range(frames_y):
        ctx.frame([(0, _use("slot", 7, [2], rng))])
    ctx.frame([(0, _use("slot", 7, [4], rng))])


@pytest.mark.parametrize("scenario,n", [(_sit_out, 63), (_sit_out, 127), (_hand_over, 63), (_hand_over, 127)])
def test_signature_only_rule_consumes_stale_words(words, rule, scenario, n):
    """The signature alone misses both cases: a tile of the returning run takes a word written 64 (128) frames earlier."""
    ctx = Context(words, SignatureOnlyRule(rule), epoch_start=1000, rng=random.Random(n))
    with pytest.raises(AssertionError, match="stale"):
        scenario(ctx, n, random.Random(n))


@pytest.mark.parametrize("scenario", [_sit_out, _hand_over])
@pytest.mark.parametrize("n", [1, 62, 63, 64, 65, 127, 128, 200])
def test_rule_zeroes_before_an_aliasing_run(words, rule, scenario, n):
    ctx = Context(words, RealRule(rule), epoch_start=1000)
    scenario(ctx, n, random.Random(n))
    # a slot's first run zeroes (its signature changes from nothing); then only the 64-frame limit does, the signatures
    # never change: slot 0 runs every frame, n + 2 times, and slot 1 returns n + 1 frames after its first run
    want = 1 + (n + 1) // 64
    if scenario is _sit_out:
        want += 1 + (1 if n + 1 >= 64 else 0)
    assert ctx.clears == want


def test_rule_across_the_30_bit_wrap(words, rule):
    """Slot order sits out across the wrap (next_epoch zeroes every array there), default order runs through it."""
    for gap in (0, 1, 62, 63, 64, 65, 127, 128):
        for start in range(EPOCH_MASK - 66, EPOCH_MASK + 1, 13):
            rng = random.Random(gap * 7 + start)
            ctx = Context(words, RealRule(rule), epoch_start=start)
            ctx.frame([(0, _use("slot", 3, [3], rng)), (1, _use("default", 0, [2, 1], rng))])
            for _ in range(gap):
                ctx.frame([(1, _use("default", 0, [rng.randint(0, 3), 1], rng))])
            for _ in range(70):
                ctx.frame([(0, _use("slot", 3, [3], rng)), (1, _use("default", 0, [rng.randint(0, 3)], rng))])


# ---- random multi-frame sequences with the real rule --------------------------------------------------------------------
GAPS = [1, 2, 5, 31, 62, 63, 64, 65, 126, 127, 128, 129, 191, 192, 200]


def _sequence(ctx, rng, n_events):
    """Random hnb_simulate frames: 1-3 batch slots, each either running an instance set (the same one, another instance of
    the same effect and slab = a re-pointed spawner row, or another effect / slab = another signature) or sitting out for a
    gap; frames with no batch at all; populations that change from run to run."""
    n_slots = rng.randint(1, 3)
    # instance sets: (order, signature, tile count per instance); several share a signature with different geometry
    uses = []
    for k in range(rng.randint(2, 5)):
        order = rng.choice(["slot", "slot", "default"])
        sig = rng.choice([5, 6, 100 + k]) if order == "slot" else 0
        uses.append((order, sig, [rng.randint(1, 5) for _ in range(rng.randint(1, 3))]))
    current = {s: rng.randrange(len(uses)) for s in range(n_slots)}
    resume_at = {s: 0 for s in range(n_slots)}
    for _ in range(n_events):
        batches = []
        for s in range(n_slots):
            if ctx.frame_no < resume_at[s]:
                continue
            r = rng.random()
            if r < 0.08:
                resume_at[s] = ctx.frame_no + (rng.choice(GAPS) if rng.random() < 0.7 else rng.randint(1, 200))
                continue
            if r < 0.2:
                current[s] = rng.randrange(len(uses))
            order, sig, tiles = uses[current[s]]
            if order == "default":                                      # default order: tiles follow the population
                tiles = [rng.randint(0, 5) for _ in tiles]
            batches.append((s, _use(order, sig, tiles, rng)))
        if not batches and rng.random() < 0.3:
            for _ in range(rng.choice(GAPS)):                           # frames with zero batches
                ctx.frame([])
        ctx.frame(batches, schedule=rng.choice(["adversarial", "adversarial", "random"]))


@pytest.mark.parametrize("seed", range(8))
def test_random_sequences_never_consume_a_stale_word(words, rule, seed):
    """Thousands of sequences in all (250 per seed): sit-outs of 1-200 frames, re-pointed spawner rows, batch slots changing
    effect or slab, empty frames, and starts near the 30-bit wrap. Every tile gets its exact exclusive prefix."""
    rng = random.Random(1000 + seed)
    clears = 0
    for _ in range(250):
        start = rng.choice([0, rng.randrange(EPOCH_MASK - 400, EPOCH_MASK + 1), rng.randrange(1, EPOCH_MASK)])
        ctx = Context(words, RealRule(rule), epoch_start=start, rng=rng)
        _sequence(ctx, rng, rng.randint(20, 60))
        clears += ctx.clears
    assert clears > 0


def test_the_same_sequences_catch_the_signature_only_rule(words, rule):
    """The random sequences are sharp enough: under the old rule some of them consume a stale word."""
    rng = random.Random(5)
    with pytest.raises(AssertionError, match="stale"):
        for _ in range(250):
            ctx = Context(words, SignatureOnlyRule(rule), epoch_start=rng.randrange(1, EPOCH_MASK), rng=rng)
            _sequence(ctx, rng, rng.randint(20, 60))
