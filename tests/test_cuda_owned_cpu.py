"""The owners of bevy_hanabi_b200/csrc/runtime/cuda_owned.h under failing CUDA calls, on the CPU.

context.cpp holds every device array, pinned block, event and stream of a context in these owners, and grows its tables
with `grow`. A CUDA call that fails throws out of the C ABI call half-way, so the owners alone decide whether anything
leaks or dangles. The header is compiled with g++ against a fake CUDA runtime that keeps host memory for device memory,
tracks every live allocation, event and stream, checks that every memset and copy stays inside a live allocation, and
fails the k-th call of a chosen function. For every grow shape context.cpp uses and every k:
  * a failed grow leaves the owner with its old block, size and contents, and releases the new block;
  * a successful grow keeps the prefix it was asked to keep, zeroes the rest, and synchronises before releasing the old
    block (an empty owner has nothing to wait for);
  * a moved-from owner releases nothing, and nothing is live once every owner has gone out of scope;
  * a borrowed stream is never destroyed.
"""
import ctypes as C
import hashlib
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "build" / "cuda_owned"
OWNED_H = ROOT / "bevy_hanabi_b200" / "csrc" / "runtime" / "cuda_owned.h"

FAKE_RUNTIME_H = r"""
#pragma once
#include <stddef.h>
typedef enum cudaError { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2 } cudaError_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
typedef struct CUstream_st* cudaStream_t;
typedef struct CUevent_st* cudaEvent_t;
cudaError_t cudaMalloc(void** p, size_t bytes);
cudaError_t cudaFree(void* p);
cudaError_t cudaMallocHost(void** p, size_t bytes);
cudaError_t cudaFreeHost(void* p);
cudaError_t cudaMemsetAsync(void* p, int value, size_t bytes, cudaStream_t st);
cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st);
cudaError_t cudaStreamSynchronize(cudaStream_t st);
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned flags);
cudaError_t cudaEventDestroy(cudaEvent_t e);
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* st, unsigned flags);
cudaError_t cudaStreamDestroy(cudaStream_t st);
"""

DRIVER = r"""
#include "cuda_owned.h"

#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <set>
#include <string>

using namespace hnb_rt;

// ---- the fake runtime ----
enum Fn { kMalloc, kMallocHost, kMemset, kMemcpy, kSync, kEventCreate, kStreamCreate, kFns };
namespace {
struct Fake {
    std::map<char*, size_t> device, host;  // live allocations and their sizes
    std::set<uintptr_t> events, streams;   // live handles
    long calls[kFns] = {};
    int fail_fn = -1;
    long fail_at = 0;
    bool injected = false;
    uintptr_t next_handle = 0x1000;
    std::string err;  // the first misuse seen
} g;

void misuse(const std::string& what) {
    if (g.err.empty()) g.err = what;
}
bool fails(Fn f) {
    if (++g.calls[f] == g.fail_at && f == g.fail_fn) return g.injected = true;
    return false;
}
void arm(int fn, long k) {
    for (long& n : g.calls) n = 0;
    g.fail_fn = fn;
    g.fail_at = k;
    g.injected = false;
}
void disarm() { g.fail_fn = -1; }
bool in_device(const void* p, size_t bytes) {
    const char* q = static_cast<const char*>(p);
    auto it = g.device.upper_bound(const_cast<char*>(q));
    if (it == g.device.begin()) return false;
    --it;
    return q >= it->first && q + bytes <= it->first + it->second;
}
cudaError_t alloc_in(std::map<char*, size_t>& live, void** p, size_t bytes) {
    char* q = static_cast<char*>(malloc(bytes ? bytes : 1));
    memset(q, 0xA5, bytes);  // not zero: zeroing is the caller's job
    live[q] = bytes;
    *p = q;
    return cudaSuccess;
}
cudaError_t free_in(std::map<char*, size_t>& live, void* p, const char* what) {
    if (!live.erase(static_cast<char*>(p))) {
        misuse(std::string(what) + " of a pointer that is not live");
        return cudaErrorInvalidValue;
    }
    free(p);
    return cudaSuccess;
}
cudaError_t create_in(std::set<uintptr_t>& live, uintptr_t* h) {
    *h = g.next_handle++;
    live.insert(*h);
    return cudaSuccess;
}
cudaError_t destroy_in(std::set<uintptr_t>& live, uintptr_t h, const char* what) {
    if (!live.erase(h)) {
        misuse(std::string(what) + " of a handle this runtime did not create, or destroyed twice");
        return cudaErrorInvalidValue;
    }
    return cudaSuccess;
}
}  // namespace

cudaError_t cudaMalloc(void** p, size_t bytes) { return fails(kMalloc) ? cudaErrorMemoryAllocation : alloc_in(g.device, p, bytes); }
cudaError_t cudaFree(void* p) { return free_in(g.device, p, "cudaFree"); }
cudaError_t cudaMallocHost(void** p, size_t bytes) { return fails(kMallocHost) ? cudaErrorMemoryAllocation : alloc_in(g.host, p, bytes); }
cudaError_t cudaFreeHost(void* p) { return free_in(g.host, p, "cudaFreeHost"); }
cudaError_t cudaMemsetAsync(void* p, int value, size_t bytes, cudaStream_t) {
    if (fails(kMemset)) return cudaErrorInvalidValue;
    if (!in_device(p, bytes)) misuse("cudaMemsetAsync outside a live device allocation");
    else memset(p, value, bytes);
    return cudaSuccess;
}
cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, cudaStream_t) {
    if (fails(kMemcpy)) return cudaErrorInvalidValue;
    if (kind != cudaMemcpyDeviceToDevice || !in_device(dst, bytes) || !in_device(src, bytes)) misuse("cudaMemcpyAsync outside live device allocations");
    else memcpy(dst, src, bytes);
    return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t) { return fails(kSync) ? cudaErrorInvalidValue : cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) {
    return fails(kEventCreate) ? cudaErrorMemoryAllocation : create_in(g.events, reinterpret_cast<uintptr_t*>(e));
}
cudaError_t cudaEventDestroy(cudaEvent_t e) { return destroy_in(g.events, reinterpret_cast<uintptr_t>(e), "cudaEventDestroy"); }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* st, unsigned) {
    return fails(kStreamCreate) ? cudaErrorMemoryAllocation : create_in(g.streams, reinterpret_cast<uintptr_t*>(st));
}
cudaError_t cudaStreamDestroy(cudaStream_t st) { return destroy_in(g.streams, reinterpret_cast<uintptr_t>(st), "cudaStreamDestroy"); }

// ---- the cases ----
namespace {
template <size_t N> struct Elem {
    unsigned char b[N];
};
const cudaStream_t kStream = reinterpret_cast<cudaStream_t>(uintptr_t(0x10));
constexpr size_t kOld = 5, kNew = 13;

unsigned char pattern(size_t byte) { return static_cast<unsigned char>(byte * 7 + 1); }

// mode 0: keep none of a filled owner, 1: keep its prefix, 2: grow an empty owner (a zero-filled allocation)
template <size_t N> std::string grow_case(int mode, int fn, long k) {
    using T = Elem<N>;
    {
        DeviceArray<T> a;
        if (mode != 2) {
            if (grow(a, kOld, 0, kStream) != cudaSuccess) return "set-up grow failed";
            for (size_t i = 0; i < kOld * N; ++i) reinterpret_cast<unsigned char*>(a.get())[i] = pattern(i);
        }
        T* const old_p = a.get();
        const size_t old_n = a.size();
        arm(fn, k);
        const cudaError_t e = grow(a, kNew, mode == 1 ? kOld : 0, kStream);
        disarm();
        const unsigned char* bytes = reinterpret_cast<const unsigned char*>(a.get());
        if (e != cudaSuccess) {
            if (!g.injected) return "grow failed with no injected failure";
            if (a.get() != old_p || a.size() != old_n) return "a failed grow changed the owner's block or size";
            for (size_t i = 0; i < old_n * N; ++i)
                if (bytes[i] != pattern(i)) return "a failed grow changed the old contents";
            if (g.device.size() != (old_p ? 1u : 0u)) return "a failed grow left its new block live";
        } else {
            if (g.injected) return "grow reported success over an injected failure";
            if (a.size() != kNew || !a.get() || a.get() == old_p) return "a grow did not install its new block";
            for (size_t i = 0; i < kNew * N; ++i)
                if (bytes[i] != (mode == 1 && i < kOld * N ? pattern(i) : 0)) return "a grow did not keep the prefix and zero the rest";
            if (g.device.size() != 1) return "a grow left the old block live";
            if (g.calls[kSync] != (old_p ? 1 : 0)) return "a grow must synchronise once before releasing an old block, and only then";
        }
        DeviceArray<T> b = std::move(a);
        if (a.get() || a.size()) return "a moved-from owner still holds a block";
        DeviceArray<T> c;
        if (c.alloc(3) != cudaSuccess) return "set-up alloc failed";
        c = std::move(b);  // releases c's own block
        if (g.device.size() != (c ? 1u : 0u)) return "move assignment did not release the target's block";
    }
    if (!g.device.empty()) return "a device allocation is live after every owner went out of scope";
    return g.err;
}

std::string handles_case(int fn, long k) {
    {
        arm(fn, k);
        PinnedBlock p;
        cudaError_t e = p.alloc(64);
        if ((e == cudaSuccess) != bool(p) || (p && p.size() != 64)) return "pinned block does not match its allocation";
        e = p.alloc(128);  // releases the first block
        if ((e == cudaSuccess) != bool(p) || g.host.size() != (p ? 1u : 0u)) return "re-allocating a pinned block kept the old one";
        Event ev;
        e = ev.create(0);
        if ((e == cudaSuccess) != (ev.get() != nullptr)) return "event does not match its creation";
        Stream owned;
        e = owned.create(1);
        if ((e == cudaSuccess) != (owned.get() != nullptr)) return "stream does not match its creation";
        Stream moved = std::move(owned);
        if (owned.get()) return "a moved-from stream still holds its handle";
        Stream borrowed;
        borrowed.borrow(reinterpret_cast<cudaStream_t>(uintptr_t(0x77)));  // not created here: destroying it is a misuse
        Stream moved_borrowed = std::move(borrowed);
        disarm();
    }
    if (!g.host.empty() || !g.events.empty() || !g.streams.empty()) return "a pinned block, event or stream is live after every owner went out of scope";
    return g.err;
}

std::string result;
void reset() {
    disarm();
    g.err.clear();
}
}  // namespace

// Returns "" when the case holds, else what went wrong. *injected: the k-th call of `fn` happened (and failed).
extern "C" const char* run_grow(int elem_bytes, int mode, int fn, long k, int* injected) {
    reset();
    switch (elem_bytes) {
        case 1: result = grow_case<1>(mode, fn, k); break;
        case 4: result = grow_case<4>(mode, fn, k); break;
        case 8: result = grow_case<8>(mode, fn, k); break;
        case 20: result = grow_case<20>(mode, fn, k); break;
        case 60: result = grow_case<60>(mode, fn, k); break;
        default: result = "no such element size";
    }
    *injected = g.injected;
    return result.c_str();
}
extern "C" const char* run_handles(int fn, long k, int* injected) {
    reset();
    result = handles_case(fn, k);
    *injected = g.injected;
    return result.c_str();
}
"""

FNS = {"cudaMalloc": 0, "cudaMallocHost": 1, "cudaMemsetAsync": 2, "cudaMemcpyAsync": 3, "cudaStreamSynchronize": 4,
       "cudaEventCreateWithFlags": 5, "cudaStreamCreateWithFlags": 6}
# Element sizes of the grown arrays of context.cpp: bytes (arena, planes, properties), words (tile prefix, batch scratch,
# event buffers, alive bits), 8 bytes (tile states, sort scratch, child infos, debug counters), draw args, metadata rows.
ELEM_BYTES = [1, 4, 8, 20, 60]
MODES = {"keep_none": 0, "keep_prefix": 1, "empty_owner": 2}


@pytest.fixture(scope="module")
def lib():
    text = DRIVER + "// " + hashlib.sha1(OWNED_H.read_bytes()).hexdigest() + "\n"
    tag = hashlib.sha1((FAKE_RUNTIME_H + text).encode()).hexdigest()[:16]
    build = OUT / tag
    so = build / "owned.so"
    if not so.exists():
        build.mkdir(parents=True, exist_ok=True)
        (build / "cuda_runtime_api.h").write_text(FAKE_RUNTIME_H)
        cpp = build / "driver.cpp"
        cpp.write_text(text)
        tmp = f"{so}.{id(text)}.tmp"
        proc = subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-Wall", "-Werror", "-I", str(build), "-I", str(OWNED_H.parent),
                               str(cpp), "-o", tmp], capture_output=True, text=True)
        assert proc.returncode == 0, proc.stderr[:4000]
        Path(tmp).replace(so)
    lib = C.CDLL(str(so))
    for fn, args in (("run_grow", [C.c_int, C.c_int, C.c_int, C.c_long, C.POINTER(C.c_int)]),
                     ("run_handles", [C.c_int, C.c_long, C.POINTER(C.c_int)])):
        getattr(lib, fn).argtypes, getattr(lib, fn).restype = args, C.c_char_p
    return lib


def every_k(run):
    """Runs the case with the k-th call failing for k = 1, 2, ... until a run makes fewer than k calls (and one with none
    failing); returns how many runs had a failure injected."""
    injected, k = C.c_int(0), 1
    while True:
        msg = run(k, C.byref(injected)).decode()
        assert msg == "", f"k={k}: {msg}"
        if not injected.value:
            return k - 1
        k += 1


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("fn", ["cudaMalloc", "cudaMemsetAsync", "cudaMemcpyAsync", "cudaStreamSynchronize"])
def test_grow_keeps_the_old_block_when_a_step_fails(lib, fn, mode):
    for elem in ELEM_BYTES:
        failures = every_k(lambda k, inj: lib.run_grow(elem, MODES[mode], FNS[fn], k, inj))
        # the calls grow makes: one allocation and one memset, a copy when it keeps a prefix, a sync when it has an old block
        expected = {"cudaMalloc": 1, "cudaMemsetAsync": 1, "cudaMemcpyAsync": 1 if mode == "keep_prefix" else 0,
                    "cudaStreamSynchronize": 0 if mode == "empty_owner" else 1}[fn]
        assert failures == expected, (elem, failures)


@pytest.mark.parametrize("fn", ["cudaMallocHost", "cudaEventCreateWithFlags", "cudaStreamCreateWithFlags"])
def test_pinned_blocks_events_and_streams_release_exactly_what_they_own(lib, fn):
    assert every_k(lambda k, inj: lib.run_handles(FNS[fn], k, inj)) >= 1
